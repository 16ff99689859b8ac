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

using namespace cupoch;

static int fails = 0;
#define EXPECT(cond)                                                          \
    do {                                                                      \
        if (!(cond)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++fails; } \
    } while (0)

static std::vector<Eigen::Vector3f> read_rows(const std::string &path) {
    std::vector<Eigen::Vector3f> rows;
    std::FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) return rows;
    float v[3];
    while (std::fread(v, sizeof(float), 3, f) == 3) rows.push_back(Eigen::Vector3f(v[0], v[1], v[2]));
    std::fclose(f);
    return rows;
}

static bool same(const Eigen::Vector3f &a, const Eigen::Vector3f &b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2]; }

static void write_rows(const std::string &path, const std::vector<Eigen::Vector3f> &rows) {
    std::FILE *f = std::fopen(path.c_str(), "wb");
    for (const auto &r : rows) {
        const float v[3] = {r[0], r[1], r[2]};
        std::fwrite(v, sizeof(float), 3, f);
    }
    std::fclose(f);
}

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
        geometry::PointCloud pcd(read_rows(dir + "/points.f32"));
        pcd.SetNormals(read_rows(dir + "/normals.f32"));
        if (pcd.IsEmpty() || !pcd.HasNormals()) return 2;
        auto out = pcd.FarthestPointDownSample((size_t)std::atol(argv[2]));
        write_rows(dir + "/out_points.f32", out->GetPoints());
        write_rows(dir + "/out_normals.f32", out->GetNormals());
    }
    if (fails) return 1;
    std::printf("facade FarthestPointDownSample: all expectations met\n");
    return 0;
}
