// VoxelGrid::CreateFromTriangleMesh[WithinBounds] and TriangleMesh::GetMinBound / GetMaxBound through the
// header-compatible facade.  Without arguments: a compile-and-link check.  With DIR: known answers (the cell-centre rule,
// an empty mesh, a rejected index), then DIR/mesh.f32 = vertices [n][3] and DIR/mesh.i32 = triangles [m][3] are
// voxelised over DIR/bounds.f32 = voxel size, min xyz, max xyz and over the mesh's own bounds; every result goes to
// DIR/out_*.  Exit code 0 = all expectations met.
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/geometry/trianglemesh.h"
#include "cupoch/geometry/voxelgrid.h"
#include "facade_check.h"

using namespace cupoch;

static bool same3(const Eigen::Vector3f &a, float x, float y, float z) { return a[0] == x && a[1] == y && a[2] == z; }

static void write_grid(const std::string &d, const std::string &name, const geometry::VoxelGrid &g) {
    const auto k = g.voxels_keys_.to_host();
    const auto c = g.voxels_colors_.to_host();
    write_file(d + "/out_" + name + "_keys.i32", k.data(), k.size() * 12);
    write_file(d + "/out_" + name + "_colors.f32", c.data(), c.size() * 12);
    const float geo[4] = {g.voxel_size_, g.origin_[0], g.origin_[1], g.origin_[2]};
    write_file(d + "/out_" + name + "_geometry.f32", geo, sizeof(geo));
}

int main(int argc, char **argv) {
    if (argc != 2) return 0;  // compile-and-link check only
    const std::string d = argv[1];
    {  // a triangle in the plane z = 0.75 vs lies in cell k_z = 0
        geometry::TriangleMesh m(std::vector<Eigen::Vector3f>{{0.1f, 0.1f, 0.375f}, {1.9f, 0.1f, 0.375f}, {0.1f, 1.9f, 0.375f}},
                                 std::vector<Eigen::Vector3i>{{0, 1, 2}});
        auto g = geometry::VoxelGrid::CreateFromTriangleMeshWithinBounds(m, 0.5f, Eigen::Vector3f(0, 0, 0), Eigen::Vector3f(2, 2, 2));
        const auto k = g->voxels_keys_.to_host();
        EXPECT(k.size() == 13);
        for (const auto &x : k) EXPECT(x[2] == 0);
        EXPECT(same3(m.GetMinBound(), 0.1f, 0.1f, 0.375f) && same3(m.GetMaxBound(), 1.9f, 1.9f, 0.375f));
        geometry::TriangleMesh empty;
        auto e = geometry::VoxelGrid::CreateFromTriangleMesh(empty, 0.5f);
        EXPECT(!e->HasVoxels() && e->voxel_size_ == 0.5f && same3(e->origin_, -0.25f, -0.25f, -0.25f));
        geometry::TriangleMesh bad(std::vector<Eigen::Vector3f>{{0, 0, 0}}, std::vector<Eigen::Vector3i>{{0, 0, 1}});
        bool threw = false;
        try {
            geometry::VoxelGrid::CreateFromTriangleMesh(bad, 0.5f);
        } catch (const std::runtime_error &) {
            threw = true;
        }
        EXPECT(threw);
    }
    const auto f = read_file<float>(d + "/mesh.f32");
    const auto t = read_file<int32_t>(d + "/mesh.i32");
    const auto b = read_file<float>(d + "/bounds.f32");
    std::vector<Eigen::Vector3i> tri(t.size() / 3);
    for (size_t i = 0; i < tri.size(); ++i) tri[i] = Eigen::Vector3i(t[3 * i], t[3 * i + 1], t[3 * i + 2]);
    geometry::TriangleMesh mesh(rows3(f), tri);
    write_grid(d, "within", *geometry::VoxelGrid::CreateFromTriangleMeshWithinBounds(mesh, b[0], Eigen::Vector3f(b[1], b[2], b[3]),
                                                                                     Eigen::Vector3f(b[4], b[5], b[6])));
    write_grid(d, "own", *geometry::VoxelGrid::CreateFromTriangleMesh(mesh, b[0]));
    return fails ? 1 : 0;
}
