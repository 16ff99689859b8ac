// TriangleMesh's edge list, filters, surface area and uniform sampling through the header-compatible facade.  Without
// arguments: a compile-and-link check.  With DIR: known answers (the reference's star mesh, MeshBase::FilterScope,
// the empty mesh's sampling error), then DIR/mesh.f32 = vertices, normals, colours [n][3] each and DIR/mesh.i32 =
// triangles [m][3] are filtered, measured and sampled; every result goes to DIR/out_*.  Exit code 0 = all expectations
// met.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/geometry/trianglemesh.h"
#include "facade_check.h"

using namespace cupoch;

static void write3(const std::string &path, const utility::device_vector<Eigen::Vector3f> &v) {
    const auto h = v.to_host();
    write_file(path, h.data(), h.size() * 12);
}

int main(int argc, char **argv) {
    if (argc != 2) return 0;  // compile-and-link check only
    const std::string d = argv[1];
    using Scope = geometry::MeshBase::FilterScope;
    {  // the reference's star: FilterSharpen(1, 1) moves every rim vertex to 4
        geometry::TriangleMesh m(std::vector<Eigen::Vector3f>{{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {-1, 0, 0}, {0, -1, 0}},
                                 std::vector<Eigen::Vector3i>{{0, 1, 2}, {0, 2, 3}, {0, 3, 4}, {0, 4, 1}});
        EXPECT(!m.HasEdgeList());
        m.ComputeEdgeList();
        EXPECT(m.HasEdgeList() && m.edge_list_.size() == 16);
        const auto v = m.FilterSharpen(1, 1.f)->vertices_.to_host();
        EXPECT(v[1][0] == 4.f && v[2][1] == 4.f && v[3][0] == -4.f && v[4][1] == -4.f && v[0][0] == 0.f);
        const auto s = m.FilterSmoothSimple(1, geometry::TriangleMesh::FilterScope::Vertex)->vertices_.to_host();
        EXPECT(s[1][0] == 0.25f);
        EXPECT(std::fabs(m.GetSurfaceArea() - 2.f) == 0.f);
        geometry::TriangleMesh empty;
        bool threw = false;
        try {
            empty.SamplePointsUniformly(100);
        } catch (const std::runtime_error &) {
            threw = true;
        }
        EXPECT(threw);
    }
    const auto f = read_file<float>(d + "/mesh.f32");
    const auto t = read_file<int32_t>(d + "/mesh.i32");
    const size_t n = f.size() / 9, m = t.size() / 3;
    std::vector<Eigen::Vector3f> v(n), vn(n), vc(n);
    for (size_t i = 0; i < n; ++i) {
        v[i] = Eigen::Vector3f(f[3 * i], f[3 * i + 1], f[3 * i + 2]);
        vn[i] = Eigen::Vector3f(f[3 * (n + i)], f[3 * (n + i) + 1], f[3 * (n + i) + 2]);
        vc[i] = Eigen::Vector3f(f[3 * (2 * n + i)], f[3 * (2 * n + i) + 1], f[3 * (2 * n + i) + 2]);
    }
    std::vector<Eigen::Vector3i> tri(m);
    for (size_t i = 0; i < m; ++i) tri[i] = Eigen::Vector3i(t[3 * i], t[3 * i + 1], t[3 * i + 2]);
    geometry::TriangleMesh mesh(v, tri);
    mesh.vertex_normals_ = vn;
    mesh.vertex_colors_ = vc;
    mesh.ComputeEdgeList();
    {
        const auto e = mesh.edge_list_.to_host();
        write_file(d + "/out_edges.i32", e.data(), e.size() * 8);
    }
    auto sh = mesh.FilterSharpen(3, 0.2f, Scope::All);
    write3(d + "/out_sharpen_v.f32", sh->vertices_);
    write3(d + "/out_sharpen_n.f32", sh->vertex_normals_);
    write3(d + "/out_sharpen_c.f32", sh->vertex_colors_);
    write3(d + "/out_simple_v.f32", mesh.FilterSmoothSimple(5, Scope::Color)->vertex_colors_);
    write3(d + "/out_laplacian_v.f32", mesh.FilterSmoothLaplacian(10, 0.5f, Scope::Vertex)->vertices_);
    auto tb = mesh.FilterSmoothTaubin(10, 0.5f, -0.53f, Scope::Normal);
    write3(d + "/out_taubin_n.f32", tb->vertex_normals_);
    write3(d + "/out_taubin_v.f32", tb->vertices_);
    utility::device_vector<float> areas;
    const float total = mesh.GetSurfaceArea(areas);
    EXPECT(total == mesh.GetSurfaceArea());
    {
        auto h = areas.to_host();
        h.push_back(total);
        write_file(d + "/out_area.f32", h.data(), h.size() * 4);
    }
    auto pc = mesh.SamplePointsUniformly(12345);
    write3(d + "/out_sample_p.f32", pc->points_);
    write3(d + "/out_sample_n.f32", pc->normals_);
    write3(d + "/out_sample_c.f32", pc->colors_);
    mesh.triangle_normals_.clear();
    auto pt = mesh.SamplePointsUniformly(777, true);
    EXPECT(mesh.HasTriangleNormals());
    write3(d + "/out_sample_tn.f32", pt->normals_);
    return fails ? 1 : 0;
}
