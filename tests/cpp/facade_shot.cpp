// registration::ComputeSHOTFeature through the header-compatible facade:
//   - an empty input gives an empty feature; missing normals and an illegal search are logged;
//   - with DIR: ComputeSHOTFeature(pcd, radius, KDTreeSearchParamRadius(radius, 100)) on DIR/points.f32 with
//     DIR/normals.f32, radius read from DIR/radius.f32; the [n][352] rows written to DIR/out_shot.f32.
// Exit code 0 = all expectations met.
#include <cstdio>
#include <string>
#include <vector>

#include "cupoch/geometry/pointcloud.h"
#include "cupoch/knn/kdtree_search_param.h"
#include "cupoch/registration/feature.h"
#include "facade_check.h"

using namespace cupoch;

int main(int argc, char **argv) {
    {
        geometry::PointCloud empty;
        auto f = registration::ComputeSHOTFeature(empty, 0.1f, knn::KDTreeSearchParamKNN(30));
        EXPECT(f->Num() == 0 && f->Dimension() == 352);
    }
    if (argc == 2) {
        const std::string dir = argv[1];
        geometry::PointCloud pcd(rows3(read_file<float>(dir + "/points.f32")));
        const std::vector<float> r = read_file<float>(dir + "/radius.f32");
        if (pcd.IsEmpty() || r.size() != 1) return 2;
        auto no_normals = registration::ComputeSHOTFeature(pcd, r[0], knn::KDTreeSearchParamRadius(r[0], 100));
        EXPECT(no_normals->Num() == pcd.points_.size());
        pcd.SetNormals(rows3(read_file<float>(dir + "/normals.f32")));
        auto bad = registration::ComputeSHOTFeature(pcd, r[0], knn::KDTreeSearchParamKNN(101));
        EXPECT(bad->Num() == pcd.points_.size());
        auto f = registration::ComputeSHOTFeature(pcd, r[0], knn::KDTreeSearchParamRadius(r[0], 100));
        EXPECT(f->Num() == pcd.points_.size() && f->Dimension() == 352 && f->data_.size() == 352 * pcd.points_.size());
        std::vector<float> h(f->data_.size());
        utility::check(cphb_memcpy_d2h(h.data(), f->data_.data(), h.size() * sizeof(float), nullptr));
        write_file(dir + "/out_shot.f32", h.data(), h.size() * sizeof(float));
    }
    if (fails) return 1;
    std::printf("facade ComputeSHOTFeature: all expectations met\n");
    return 0;
}
