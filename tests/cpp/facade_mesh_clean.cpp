// TriangleMesh::RemoveDuplicatedVertices / RemoveDuplicatedTriangles / RemoveDegenerateTriangles /
// RemoveUnreferencedVertices, GetSelfIntersectingTriangles and + / += through the header-compatible facade.  Without
// arguments: a compile-and-link check.  With DIR: known answers (a weld, a rejected index that changes nothing), then
// DIR/a.f32 + DIR/a.i32 (vertices, triangles) with DIR/a_n.f32, DIR/a_c.f32, DIR/a_tn.f32 (vertex normals, colours,
// triangle normals) and DIR/b.f32 + DIR/b.i32 are read; the cleanup chain of a, the self-intersections of b and of a + b,
// and a += b go to DIR/out_*.  Exit code 0 = all expectations met.
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/geometry/trianglemesh.h"
#include "facade_check.h"

using namespace cupoch;

static std::vector<Eigen::Vector3i> rows3i(const std::vector<int32_t> &t) {
    std::vector<Eigen::Vector3i> r(t.size() / 3);
    for (size_t i = 0; i < r.size(); ++i) r[i] = Eigen::Vector3i(t[3 * i], t[3 * i + 1], t[3 * i + 2]);
    return r;
}

template <class T>
static void dump(const std::string &path, const utility::device_vector<T> &v) {
    const auto h = v.to_host();
    write_file(path, h.data(), h.size() * sizeof(T));
}

static void dump_mesh(const std::string &d, const std::string &name, const geometry::TriangleMesh &m) {
    dump(d + "/out_" + name + "_v.f32", m.vertices_);
    dump(d + "/out_" + name + "_t.i32", m.triangles_);
    dump(d + "/out_" + name + "_n.f32", m.vertex_normals_);
    dump(d + "/out_" + name + "_c.f32", m.vertex_colors_);
    dump(d + "/out_" + name + "_tn.f32", m.triangle_normals_);
    dump(d + "/out_" + name + "_e.i32", m.edge_list_);
}

int main(int argc, char **argv) {
    if (argc != 2) return 0;  // compile-and-link check only
    const std::string d = argv[1];
    {  // two triangles sharing an edge by position only: welding merges 6 vertices into 4
        geometry::TriangleMesh m(std::vector<Eigen::Vector3f>{{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {1, 0, 0}, {0, 1, 0}, {1, 1, 0}},
                                 std::vector<Eigen::Vector3i>{{0, 1, 2}, {3, 5, 4}});
        m.RemoveDuplicatedVertices();
        EXPECT(m.vertices_.size() == 4);
        const auto t = m.triangles_.to_host();
        EXPECT(t[0][0] == 0 && t[0][1] == 2 && t[0][2] == 1 && t[1][0] == 2 && t[1][1] == 3 && t[1][2] == 1);
        geometry::TriangleMesh bad(std::vector<Eigen::Vector3f>{{0, 0, 0}}, std::vector<Eigen::Vector3i>{{0, 0, 1}});
        bool threw = false;
        try {
            bad.RemoveDegenerateTriangles();
        } catch (const std::runtime_error &) {
            threw = true;
        }
        EXPECT(threw && bad.triangles_.size() == 1);
    }
    geometry::TriangleMesh a(rows3(read_file<float>(d + "/a.f32")), rows3i(read_file<int32_t>(d + "/a.i32")));
    a.vertex_normals_ = rows3(read_file<float>(d + "/a_n.f32"));
    a.vertex_colors_ = rows3(read_file<float>(d + "/a_c.f32"));
    a.triangle_normals_ = rows3(read_file<float>(d + "/a_tn.f32"));
    a.ComputeEdgeList();
    geometry::TriangleMesh b(rows3(read_file<float>(d + "/b.f32")), rows3i(read_file<int32_t>(d + "/b.i32")));
    const geometry::TriangleMesh sum = a + b;
    geometry::TriangleMesh acc = a;
    acc += b;
    dump_mesh(d, "sum", sum);
    dump_mesh(d, "acc", acc);
    a.RemoveDuplicatedVertices();
    dump_mesh(d, "dv", a);
    a.RemoveDuplicatedTriangles();
    dump_mesh(d, "dt", a);
    a.RemoveDegenerateTriangles();
    dump_mesh(d, "dg", a);
    a.RemoveUnreferencedVertices();
    dump_mesh(d, "ur", a);
    dump(d + "/out_self_b.i32", b.GetSelfIntersectingTriangles());
    return fails ? 1 : 0;
}
