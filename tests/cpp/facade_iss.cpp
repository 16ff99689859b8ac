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

static void write_bytes(const std::string &path, const void *p, size_t bytes) {
    std::FILE *f = std::fopen(path.c_str(), "wb");
    std::fwrite(p, 1, bytes, f);
    std::fclose(f);
}

static void write_rows(const std::string &path, const std::vector<Eigen::Vector3f> &rows) {
    std::vector<float> flat;
    for (const auto &r : rows) flat.insert(flat.end(), {r[0], r[1], r[2]});
    write_bytes(path, flat.data(), flat.size() * sizeof(float));
}

int main(int argc, char **argv) {
    {
        geometry::PointCloud empty;
        auto res = geometry::keypoint::ComputeISSKeypoints(empty);
        EXPECT(std::get<0>(res)->IsEmpty() && std::get<1>(res)->empty());
    }
    if (argc == 2) {
        const std::string dir = argv[1];
        geometry::PointCloud pcd(read_rows(dir + "/points.f32"));
        pcd.SetNormals(read_rows(dir + "/normals.f32"));
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
        write_rows(dir + "/out_points.f32", out.GetPoints());
        write_rows(dir + "/out_normals.f32", out.GetNormals());
        write_bytes(dir + "/out_mask.u8", h.data(), h.size());
    }
    if (fails) return 1;
    std::printf("facade ComputeISSKeypoints: all expectations met\n");
    return 0;
}
