// UniformTSDFVolume::ExtractTriangleMesh and TriangleMesh through the header-compatible facade.  Without arguments: a
// compile-and-link check.  With DIR: known answers (a mesh built from arrays, its normals, an unreferenced vertex and a
// bad index), then from DIR/params.f32 = {w, h, fx, fy, cx, cy, frames, length, resolution, sdf_trunc, extrinsics
// row-major [frames][16]}, DIR/depth.u16 [frames][h][w] and DIR/color.u8 [frames][h][w][3] an RGB8 volume integrates
// every frame (CreateFromColorAndDepth with depth_scale 1000, depth_trunc 100, no intensity conversion); its mesh
// (through the TSDFVolume base) and its vertex normals are written to DIR/out_*.  Exit code 0 = all expectations met.
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/camera/pinhole_camera_intrinsic.h"
#include "cupoch/geometry/rgbdimage.h"
#include "cupoch/geometry/trianglemesh.h"
#include "cupoch/integration/tsdfvolume.h"
#include "cupoch/integration/uniform_tsdfvolume.h"
#include "facade_check.h"

using namespace cupoch;

template <class T>
static void write3(const std::string &path, const utility::device_vector<T> &v) {
    const auto h = v.to_host();
    write_file(path, h.data(), h.size() * 12);
}
static geometry::Image image(const void *data, int w, int h, int ch, int bpc) {
    geometry::Image im;
    im.Prepare(w, h, ch, bpc);
    const uint8_t *b = static_cast<const uint8_t *>(data);
    im.data_ = std::vector<uint8_t>(b, b + (size_t)w * h * ch * bpc);
    return im;
}

int main(int argc, char **argv) {
    if (argc != 2) return 0;  // compile-and-link check only
    const std::string d = argv[1];
    using integration::TSDFVolumeColorType;
    {  // known answers: three right triangles at the origin, vertex 2 in none of them
        geometry::TriangleMesh m(std::vector<Eigen::Vector3f>{{0, 0, 0}, {1, 0, 0}, {5, 5, 5}, {0, 1, 0}, {0, 0, 1}},
                                 std::vector<Eigen::Vector3i>{{0, 1, 3}, {0, 3, 4}, {0, 4, 1}});
        EXPECT(m.HasVertices() && m.HasTriangles() && !m.HasTriangleNormals() && !m.HasVertexNormals());
        m.ComputeVertexNormals();
        EXPECT(m.HasTriangleNormals() && m.HasVertexNormals());
        const auto tn = m.triangle_normals_.to_host();
        EXPECT(tn[0][2] == 1.f && tn[1][0] == 1.f && tn[2][1] == 1.f);  // unnormalised, each already of unit length
        const auto vn = m.vertex_normals_.to_host();
        EXPECT(vn[2][0] == 0.f && vn[2][1] == 0.f && vn[2][2] == 0.f);
        EXPECT(vn[1][0] == 0.f && vn[1][1] == vn[1][2] && vn[1][1] > 0.707f && vn[1][1] < 0.7072f);
        geometry::TriangleMesh bad(std::vector<Eigen::Vector3f>{{0, 0, 0}}, std::vector<Eigen::Vector3i>{{0, 0, 1}});
        bool threw = false;
        try {
            bad.ComputeTriangleNormals();
        } catch (const std::runtime_error &) {
            threw = true;
        }
        EXPECT(threw);
    }
    const auto prm = read_file<float>(d + "/params.f32");
    const int w = (int)prm[0], h = (int)prm[1], frames = (int)prm[6];
    const camera::PinholeCameraIntrinsic K(w, h, prm[2], prm[3], prm[4], prm[5]);
    const auto depth = read_file<uint16_t>(d + "/depth.u16");
    const auto color = read_file<uint8_t>(d + "/color.u8");
    integration::UniformTSDFVolume vol(prm[7], (int)prm[8], prm[9], TSDFVolumeColorType::RGB8);
    for (int f = 0; f < frames; ++f) {
        auto im = geometry::RGBDImage::CreateFromColorAndDepth(image(color.data() + (size_t)f * w * h * 3, w, h, 3, 1),
                                                               image(depth.data() + (size_t)f * w * h, w, h, 1, 2), 1000.f, 100.f, false);
        vol.Integrate(*im, K, utility::from_row_major(prm.data() + 10 + 16 * f));
    }
    integration::TSDFVolume &base = vol;
    auto mesh = base.ExtractTriangleMesh();
    EXPECT(mesh->HasVertexColors() && mesh->HasTriangles() && mesh->triangles_.size() > 100);
    mesh->ComputeVertexNormals();
    EXPECT(mesh->HasVertexNormals() && mesh->HasTriangleNormals());
    write3(d + "/out_vertices.f32", mesh->vertices_);
    write3(d + "/out_vertex_colors.f32", mesh->vertex_colors_);
    write3(d + "/out_triangles.i32", mesh->triangles_);
    write3(d + "/out_triangle_normals.f32", mesh->triangle_normals_);
    write3(d + "/out_vertex_normals.f32", mesh->vertex_normals_);
    vol.Reset();
    auto empty = vol.ExtractTriangleMesh();
    EXPECT(empty->IsEmpty() && !empty->HasTriangles());
    return fails ? 1 : 0;
}
