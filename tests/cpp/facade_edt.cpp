// geometry::DistanceTransform through the header-compatible facade.  With DIR:
//   - resolution 0 and 1025 throw;
//   - ComputeEDT from a VoxelGrid of another voxel size is logged and leaves the grid unchanged;
//   - ComputeEDT(DIR/cells.i32 as [n][3] grid cells) on a DistanceTransform(DIR/params.f32 = {voxel_size, resolution,
//     ox, oy, oz}); GetDistances and GetVoxel of DIR/queries.f32 are written to DIR/out_dist.f32 and DIR/out_voxel.i32
//     ({found, x, y, z, state, distance bits} per query).
// Exit code 0 = all expectations met.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "cupoch/geometry/distancetransform.h"
#include "cupoch/geometry/voxelgrid.h"

using namespace cupoch;

static int fails = 0;
#define EXPECT(cond)                                                          \
    do {                                                                      \
        if (!(cond)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++fails; } \
    } while (0)

template <class T>
static std::vector<T> read_all(const std::string &path) {
    std::vector<T> v;
    std::FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) return v;
    T x;
    while (std::fread(&x, sizeof(T), 1, f) == 1) v.push_back(x);
    std::fclose(f);
    return v;
}

static void write_bytes(const std::string &path, const void *p, size_t bytes) {
    std::FILE *f = std::fopen(path.c_str(), "wb");
    std::fwrite(p, 1, bytes, f);
    std::fclose(f);
}

static bool throws_for(size_t res) {
    try {
        geometry::DistanceTransform dt(1.0f, res);
    } catch (const std::runtime_error &) {
        return true;
    }
    return false;
}

int main(int argc, char **argv) {
    if (argc != 2) return 0;  // compile-and-link check only
    const std::string dir = argv[1];
    const std::vector<float> prm = read_all<float>(dir + "/params.f32");
    const std::vector<int32_t> c = read_all<int32_t>(dir + "/cells.i32");
    const std::vector<float> q = read_all<float>(dir + "/queries.f32");
    if (prm.size() != 5) return 2;
    EXPECT(throws_for(0) && throws_for(1025));

    geometry::DistanceTransform dt(prm[0], (size_t)prm[1], Eigen::Vector3f(prm[2], prm[3], prm[4]));
    std::vector<Eigen::Vector3i> cells;
    for (size_t i = 0; i + 2 < c.size(); i += 3) cells.push_back(Eigen::Vector3i(c[i], c[i + 1], c[i + 2]));
    dt.ComputeEDT(utility::device_vector<Eigen::Vector3i>(cells));

    geometry::VoxelGrid other;  // another voxel size: logged, nothing changes
    other.voxel_size_ = prm[0] * 2.f;
    other.voxels_keys_ = std::vector<Eigen::Vector3i>(1, Eigen::Vector3i(0, 0, 0));
    dt.ComputeEDT(other);

    std::vector<Eigen::Vector3f> queries;
    for (size_t i = 0; i + 2 < q.size(); i += 3) queries.push_back(Eigen::Vector3f(q[i], q[i + 1], q[i + 2]));
    const std::vector<float> d = dt.GetDistances(utility::device_vector<Eigen::Vector3f>(queries))->to_host();
    EXPECT(d.size() == queries.size());
    if (!queries.empty()) EXPECT(dt.GetDistance(queries[0]) == d[0]);
    write_bytes(dir + "/out_dist.f32", d.data(), d.size() * sizeof(float));

    std::vector<int32_t> vox;
    for (const auto &p : queries) {
        auto r = dt.GetVoxel(p);
        const geometry::DistanceVoxel &v = std::get<1>(r);
        EXPECT(v.IsNotSite() == ((v.state_ & geometry::DistanceVoxel::NotSite) != 0) && !v.CheckHasNext());
        int32_t bits;
        std::memcpy(&bits, &v.distance_, 4);
        vox.insert(vox.end(), {std::get<0>(r) ? 1 : 0, v.nearest_index_[0], v.nearest_index_[1], v.nearest_index_[2], (int32_t)v.state_, bits});
    }
    write_bytes(dir + "/out_voxel.i32", vox.data(), vox.size() * sizeof(int32_t));
    if (fails) return 1;
    std::printf("facade DistanceTransform: all expectations met\n");
    return 0;
}
