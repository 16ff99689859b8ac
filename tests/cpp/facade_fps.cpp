// PointCloud::FarthestPointDownSample through the header-compatible facade:
//   - the shortcuts of pointcloud.cu:301-338: 0 samples -> empty, n -> a copy in the original order, more than n ->
//     logged, the loop runs anyway; an empty cloud asked for samples stays empty;
//   - with DIR K: FarthestPointDownSample(K) on DIR/points.f32 (with DIR/normals.f32), the picked points and normals
//     written to DIR/out_points.f32 and DIR/out_normals.f32 for comparison with the oracle.
// Exit code 0 = all expectations met.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "cupoch/geometry/pointcloud.h"
#include "facade_check.h"

using namespace cupoch;

static bool same(const Eigen::Vector3f &a, const Eigen::Vector3f &b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2]; }

int main(int argc, char **argv) {
    {
        std::vector<Eigen::Vector3f> pts;
        for (int i = 0; i < 10; ++i) pts.push_back(Eigen::Vector3f((float)i, (float)(i * i % 7), 0.5f * (float)i));
        geometry::PointCloud pcd(pts);
        EXPECT(pcd.FarthestPointDownSample(0)->IsEmpty());
        auto all = pcd.FarthestPointDownSample(pts.size())->GetPoints();
        EXPECT(all.size() == pts.size());
        for (size_t i = 0; i < all.size() && i < pts.size(); ++i) EXPECT(same(all[i], pts[i]));
        auto two = pcd.FarthestPointDownSample(2)->GetPoints();  // index 0, then the farthest from it: (9, 4, 4.5)
        EXPECT(two.size() == 2 && same(two[0], pts[0]) && same(two[1], pts[9]));
        auto more = pcd.FarthestPointDownSample(pts.size() + 5)->GetPoints();  // logged; the last five repeat index 0
        EXPECT(more.size() == pts.size() + 5 && same(more.back(), pts[0]));
        geometry::PointCloud empty;
        EXPECT(empty.FarthestPointDownSample(3)->IsEmpty());
    }
    if (argc == 3) {
        const std::string dir = argv[1];
        geometry::PointCloud pcd(rows3(read_file<float>(dir + "/points.f32")));
        pcd.SetNormals(rows3(read_file<float>(dir + "/normals.f32")));
        if (pcd.IsEmpty() || !pcd.HasNormals()) return 2;
        auto out = pcd.FarthestPointDownSample((size_t)std::atol(argv[2]));
        const std::vector<float> p = rows3(out->GetPoints()), n = rows3(out->GetNormals());
        write_file(dir + "/out_points.f32", p.data(), p.size() * sizeof(float));
        write_file(dir + "/out_normals.f32", n.data(), n.size() * sizeof(float));
    }
    if (fails) return 1;
    std::printf("facade FarthestPointDownSample: all expectations met\n");
    return 0;
}
