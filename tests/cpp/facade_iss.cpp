// geometry::keypoint::ComputeISSKeypoints through the header-compatible facade:
//   - an empty input and an illegal max_neighbors are logged and give empty results;
//   - with DIR: ComputeISSKeypoints with the reference's defaults on DIR/points.f32 (with DIR/normals.f32), the keypoints,
//     their normals and the mask written to DIR/out_points.f32, DIR/out_normals.f32 and DIR/out_mask.u8.
// Exit code 0 = all expectations met.
#include <cstdio>
#include <string>
#include <vector>

#include "cupoch/geometry/keypoint.h"
#include "cupoch/geometry/pointcloud.h"
#include "facade_check.h"

using namespace cupoch;

int main(int argc, char **argv) {
    {
        geometry::PointCloud empty;
        auto res = geometry::keypoint::ComputeISSKeypoints(empty);
        EXPECT(std::get<0>(res)->IsEmpty() && std::get<1>(res)->empty());
    }
    if (argc == 2) {
        const std::string dir = argv[1];
        geometry::PointCloud pcd(rows3(read_file<float>(dir + "/points.f32")));
        pcd.SetNormals(rows3(read_file<float>(dir + "/normals.f32")));
        if (pcd.IsEmpty() || !pcd.HasNormals()) return 2;
        auto bad = geometry::keypoint::ComputeISSKeypoints(pcd, 0.f, 0.f, 0.975f, 0.975f, 5, 257);
        EXPECT(std::get<0>(bad)->IsEmpty() && std::get<1>(bad)->empty());
        auto res = geometry::keypoint::ComputeISSKeypoints(pcd);
        const auto &out = *std::get<0>(res);
        const auto &mask = *std::get<1>(res);
        EXPECT(mask.size() == pcd.points_.size());
        std::vector<unsigned char> h(mask.size());
        if (!h.empty()) utility::check(cphb_memcpy_d2h(h.data(), mask.data(), h.size(), nullptr));
        size_t m = 0;
        for (unsigned char b : h) m += b;
        EXPECT(m == out.points_.size() && out.HasNormals());
        const std::vector<float> p = rows3(out.GetPoints()), n = rows3(out.GetNormals());
        write_file(dir + "/out_points.f32", p.data(), p.size() * sizeof(float));
        write_file(dir + "/out_normals.f32", n.data(), n.size() * sizeof(float));
        write_file(dir + "/out_mask.u8", h.data(), h.size());
    }
    if (fails) return 1;
    std::printf("facade ComputeISSKeypoints: all expectations met\n");
    return 0;
}
