// facade_smoke.cpp -- exercises the header-compatible C++ facade (include/cupoch/...) the way
// cupoch's own examples/tests do (examples/cpp/registration.cpp:42-47, tests/knn/kdtree_flann.cpp).
// usage: facade_smoke <dir>   reads src.f32 tgt.f32 tgt_nrm.f32 (n x 3 float32), writes results.
#include <cstdio>
#include <string>
#include <vector>

#include "cupoch/geometry/pointcloud.h"
#include "cupoch/knn/kdtree_flann.h"
#include "cupoch/registration/registration.h"
#include "facade_check.h"

using namespace cupoch;

// a user-defined estimator: forces the generic (virtual-dispatch) loop, delegating to point-to-plane
class MyEstimation : public registration::TransformationEstimation {
public:
    registration::TransformationEstimationType GetTransformationEstimationType() const override {
        return registration::TransformationEstimationType::Unspecified;
    }
    float ComputeRMSE(const geometry::PointCloud &s, const geometry::PointCloud &t,
                      const registration::CorrespondenceSet &c) const override { return inner_.ComputeRMSE(s, t, c); }
    Eigen::Matrix4f ComputeTransformation(const geometry::PointCloud &s, const geometry::PointCloud &t,
                                          const registration::CorrespondenceSet &c) const override {
        ++calls;
        return inner_.ComputeTransformation(s, t, c);
    }
    mutable int calls = 0;

private:
    registration::TransformationEstimationPointToPlane inner_;
};

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    const std::string dir = argv[1];
    const auto src = rows3(read_file<float>(dir + "/src.f32")), tgt = rows3(read_file<float>(dir + "/tgt.f32")),
               tgt_nrm = rows3(read_file<float>(dir + "/tgt_nrm.f32"));
    if (src.empty() || tgt.empty() || tgt_nrm.empty()) {
        fprintf(stderr, "missing or empty input in %s\n", dir.c_str());
        return 2;
    }
    geometry::PointCloud source(src), target(tgt);
    target.SetNormals(tgt_nrm);

    // KDTreeFlann::SearchRadius / SearchKNN on device vectors
    knn::KDTreeFlann tree(target.points_);
    utility::device_vector<int> idx;
    utility::device_vector<float> d2;
    int k = tree.SearchRadius(source.points_, 0.03f, 1, idx, d2);
    auto hidx = idx.to_host();
    write_file(dir + "/radius_idx.i32", hidx.data(), hidx.size() * 4);
    std::vector<int> hi;
    std::vector<float> hd;
    int k1 = tree.SearchKNN(source.GetPoints()[0], 5, hi, hd);
    printf("search: k=%d single-query k=%d\n", k, k1);

    // RegistrationICP: fused path and the generic virtual loop must agree
    registration::ICPConvergenceCriteria crit(0.f, 0.f, 6);
    auto fused = registration::RegistrationICP(source, target, 0.03f, Eigen::Matrix4f::Identity(),
                                               registration::TransformationEstimationPointToPlane(), crit);
    MyEstimation mine;
    auto generic = registration::RegistrationICP(source, target, 0.03f, Eigen::Matrix4f::Identity(), mine, crit);
    float T[32];
    utility::to_row_major(fused.transformation_, T);
    utility::to_row_major(generic.transformation_, T + 16);
    write_file(dir + "/T.f32", T, sizeof(T));
    auto corr = fused.GetCorrespondenceSet();
    write_file(dir + "/corr.i32", corr.data(), corr.size() * 8);
    float fr[4] = {fused.fitness_, fused.inlier_rmse_, generic.fitness_, generic.inlier_rmse_};
    write_file(dir + "/fit.f32", fr, sizeof(fr));
    printf("icp: fitness %.4f rmse %.6f corr %zu | generic calls %d fitness %.4f\n", fused.fitness_, fused.inlier_rmse_,
           corr.size(), mine.calls, generic.fitness_);

    auto down = target.VoxelDownSample(0.05f);
    printf("voxel: %zu -> %zu (normals %d)\n", target.points_.size(), down->points_.size(), (int)down->HasNormals());
    auto ev = registration::EvaluateRegistration(source, target, 0.03f, fused.transformation_);
    printf("evaluate: fitness %.4f\n", ev.fitness_);
    return 0;
}
