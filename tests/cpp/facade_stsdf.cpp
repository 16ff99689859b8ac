// ScalableTSDFVolume through the header-compatible facade.  Without arguments: a compile-and-link check.  With DIR: the
// argument errors, then from DIR/params.f32 = {w, h, fx, fy, cx, cy, frames, voxel_length, sdf_trunc, extrinsics
// row-major [frames][16]}, DIR/depth.u16 [frames][h][w] and DIR/color.u8 [frames][h][w][3] an RGB8 volume (stride 4,
// map_size 1) integrates every frame (CreateFromColorAndDepth with depth_scale 1000, depth_trunc 4, no intensity
// conversion); ExtractPointCloud and ExtractVoxelPointCloud go to DIR/out_*.  Exit code 0 = all expectations met.
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/camera/pinhole_camera_intrinsic.h"
#include "cupoch/geometry/rgbdimage.h"
#include "cupoch/integration/scalable_tsdfvolume.h"
#include "facade_check.h"

using namespace cupoch;

static void write3(const std::string &path, const utility::device_vector<Eigen::Vector3f> &v) {
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
template <class F>
static bool throws(F f) {
    try {
        f();
    } catch (const std::runtime_error &) {
        return true;
    }
    return false;
}

int main(int argc, char **argv) {
    if (argc != 2) return 0;  // compile-and-link check only
    const std::string d = argv[1];
    using integration::TSDFVolumeColorType;
    EXPECT(throws([] { integration::ScalableTSDFVolume v(0.f, 0.04f, TSDFVolumeColorType::NoColor); }));
    EXPECT(throws([] { integration::ScalableTSDFVolume v(0.01f, 0.04f, TSDFVolumeColorType::NoColor, 0); }));
    const auto prm = read_file<float>(d + "/params.f32");
    const int w = (int)prm[0], h = (int)prm[1], frames = (int)prm[6];
    const camera::PinholeCameraIntrinsic K(w, h, prm[2], prm[3], prm[4], prm[5]);
    const auto depth = read_file<uint16_t>(d + "/depth.u16");
    const auto color = read_file<uint8_t>(d + "/color.u8");
    integration::ScalableTSDFVolume vol(prm[7], prm[8], TSDFVolumeColorType::RGB8, 4, 1);
    EXPECT(vol.volume_unit_length_ == prm[7] * 16.0f && vol.depth_sampling_stride_ == 4);
    for (int f = 0; f < frames; ++f) {
        auto im = geometry::RGBDImage::CreateFromColorAndDepth(image(color.data() + (size_t)f * w * h * 3, w, h, 3, 1),
                                                               image(depth.data() + (size_t)f * w * h, w, h, 1, 2), 1000.f, 4.f, false);
        vol.Integrate(*im, K, utility::from_row_major(prm.data() + 9 + 16 * f));
    }
    EXPECT(vol.UnitCount() > 10);
    EXPECT(throws([&] { vol.ExtractTriangleMesh(); }));
    auto pc = vol.ExtractPointCloud();
    EXPECT(pc->HasNormals() && pc->HasColors() && pc->points_.size() > 100);
    write3(d + "/out_points.f32", pc->points_);
    write3(d + "/out_normals.f32", pc->normals_);
    write3(d + "/out_colors.f32", pc->colors_);
    auto vp = vol.ExtractVoxelPointCloud();
    write3(d + "/out_vpoints.f32", vp->points_);
    write3(d + "/out_vcolors.f32", vp->colors_);
    vol.Reset();
    EXPECT(vol.UnitCount() == 0 && vol.ExtractPointCloud()->points_.size() == 0);
    return fails ? 1 : 0;
}
