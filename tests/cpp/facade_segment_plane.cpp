// PointCloud::SegmentPlane through the header-compatible facade:
//   - the reference's known-answer test (tests/geometry/pointcloud.cpp:659-673), written as it is written there;
//   - with DIR SEED THR T: srand(SEED), SegmentPlane(THR, 3, T) on DIR/points.f32, plane and inliers written to
//     DIR/plane.f32 and DIR/inliers.i64 for comparison with the oracle.
// Exit code 0 = all expectations met.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <tuple>
#include <vector>

#include "cupoch/geometry/pointcloud.h"

using namespace cupoch;

static int fails = 0;
#define EXPECT(cond)                                                          \
    do {                                                                      \
        if (!(cond)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++fails; } \
    } while (0)

int main(int argc, char **argv) {
    {   // SegmentPlaneKnownPlane
        std::vector<Eigen::Vector3f> ref_points;
        ref_points.push_back(Eigen::Vector3f(1.0f, 1.0f, -1.0f));
        ref_points.push_back(Eigen::Vector3f(2.0f, 2.0f, -5.0f));
        ref_points.push_back(Eigen::Vector3f(-1.0f, -1.0f, 1.0f));
        ref_points.push_back(Eigen::Vector3f(-2.0f, -2.0f, 3.0f));
        ref_points.push_back(Eigen::Vector3f(10.0f, 10.0f, -21.0f));
        geometry::PointCloud pcd;
        pcd.SetPoints(ref_points);
        Eigen::Vector4f plane_model;
        utility::device_vector<size_t> inliers;
        std::tie(plane_model, inliers) = pcd.SegmentPlane(0.01f, 3, 10);
        auto sel = pcd.SelectByIndex(inliers)->GetPoints();
        EXPECT(sel.size() == ref_points.size());
        for (size_t i = 0; i < sel.size() && i < ref_points.size(); ++i)
            EXPECT(sel[i][0] == ref_points[i][0] && sel[i][1] == ref_points[i][1] && sel[i][2] == ref_points[i][2]);
        // guards: logged, zero plane, no inliers
        std::tie(plane_model, inliers) = pcd.SegmentPlane(0.01f, 2, 10);
        EXPECT(inliers.empty() && plane_model[0] == 0.f && plane_model[3] == 0.f);
        std::tie(plane_model, inliers) = pcd.SegmentPlane(0.01f, 6, 10);
        EXPECT(inliers.empty());
    }
    if (argc == 5) {
        const std::string dir = argv[1];
        std::FILE *f = std::fopen((dir + "/points.f32").c_str(), "rb");
        if (!f) return 2;
        std::vector<Eigen::Vector3f> pts;
        float v[3];
        while (std::fread(v, sizeof(float), 3, f) == 3) pts.push_back(Eigen::Vector3f(v[0], v[1], v[2]));
        std::fclose(f);
        geometry::PointCloud pcd(pts);
        std::srand((unsigned)std::atoi(argv[2]));
        Eigen::Vector4f plane;
        utility::device_vector<size_t> inliers;
        std::tie(plane, inliers) = pcd.SegmentPlane((float)std::atof(argv[3]), 3, (size_t)std::atoi(argv[4]));
        float h[4] = {plane[0], plane[1], plane[2], plane[3]};
        std::vector<size_t> idx = inliers.to_host();
        std::vector<long long> out(idx.begin(), idx.end());
        f = std::fopen((dir + "/plane.f32").c_str(), "wb");
        std::fwrite(h, sizeof(float), 4, f);
        std::fclose(f);
        f = std::fopen((dir + "/inliers.i64").c_str(), "wb");
        if (!out.empty()) std::fwrite(out.data(), sizeof(long long), out.size(), f);
        std::fclose(f);
    }
    if (fails) return 1;
    std::printf("facade SegmentPlane: all expectations met\n");
    return 0;
}
