// UniformTSDFVolume and RGBDImage through the header-compatible facade.  Without arguments: a compile-and-link check.
// With DIR: known answers (PrimeSenseDefault, the argument errors, Reset), then from DIR/params.f32 =
// {w, h, fx, fy, cx, cy, frames, length, resolution, sdf_trunc, extrinsics row-major [frames][16]}, DIR/depth.u16
// [frames][h][w] and DIR/color.u8 [frames][h][w][3] an RGB8 volume integrates every frame (CreateFromColorAndDepth with
// depth_scale 1000, depth_trunc 100, no intensity conversion) and ExtractPointCloud, ExtractVoxelPointCloud,
// ExtractVoxelGrid and Raycast of frame 0 (both project_valid_depth_only values) are written to DIR/out_*.  Exit code
// 0 = all expectations met.
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/camera/pinhole_camera_intrinsic.h"
#include "cupoch/geometry/rgbdimage.h"
#include "cupoch/integration/tsdfvolume.h"
#include "cupoch/integration/uniform_tsdfvolume.h"
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
    {  // known answers
        camera::PinholeCameraIntrinsic ps(camera::PinholeCameraIntrinsicParameters::PrimeSenseDefault);
        EXPECT(ps.width_ == 640 && ps.height_ == 480 && ps.GetFocalLength().first == 525.f && ps.GetPrincipalPoint().second == 239.5f);
        EXPECT(throws([] { integration::UniformTSDFVolume v(2.f, 1, 0.1f, TSDFVolumeColorType::NoColor); }));
        EXPECT(throws([] { integration::UniformTSDFVolume v(2.f, 64, 0.f, TSDFVolumeColorType::NoColor); }));
        const std::vector<uint16_t> dd = {1999, 2000, 2499, 2500};
        const std::vector<uint8_t> cc(4, 0);
        auto im = geometry::RGBDImage::CreateFromColorAndDepth(image(cc.data(), 4, 1, 1, 1), image(dd.data(), 4, 1, 1, 2), 1000.f, 2.5f);
        const auto bytes = im->depth_.data_.to_host();
        float got[4];
        std::memcpy(got, bytes.data(), 16);
        EXPECT(got[0] == 1999.f / 1000.f && got[1] == 0.f && got[2] == 0.f && got[3] == 0.f);  // int(2.5) = 2 m
        EXPECT(throws([&] { geometry::RGBDImage::CreateFromColorAndDepth(image(cc.data(), 2, 2, 1, 1), image(dd.data(), 4, 1, 1, 2)); }));
    }
    const auto prm = read_file<float>(d + "/params.f32");
    const int w = (int)prm[0], h = (int)prm[1], frames = (int)prm[6];
    const camera::PinholeCameraIntrinsic K(w, h, prm[2], prm[3], prm[4], prm[5]);
    const auto depth = read_file<uint16_t>(d + "/depth.u16");
    const auto color = read_file<uint8_t>(d + "/color.u8");
    integration::UniformTSDFVolume vol(prm[7], (int)prm[8], prm[9], TSDFVolumeColorType::RGB8);
    EXPECT(vol.voxel_length_ == prm[7] / (float)(int)prm[8] && vol.voxel_num_ == (size_t)prm[8] * (size_t)prm[8] * (size_t)prm[8]);
    std::vector<Eigen::Matrix4f> E(frames);
    for (int f = 0; f < frames; ++f) {
        E[f] = utility::from_row_major(prm.data() + 10 + 16 * f);
        auto im = geometry::RGBDImage::CreateFromColorAndDepth(image(color.data() + (size_t)f * w * h * 3, w, h, 3, 1),
                                                               image(depth.data() + (size_t)f * w * h, w, h, 1, 2), 1000.f, 100.f, false);
        vol.Integrate(*im, K, E[f]);
    }
    auto pc = vol.ExtractPointCloud();
    EXPECT(pc->HasNormals() && pc->HasColors() && pc->points_.size() > 100);
    write3(d + "/out_points.f32", pc->points_);
    write3(d + "/out_normals.f32", pc->normals_);
    write3(d + "/out_colors.f32", pc->colors_);
    auto vp = vol.ExtractVoxelPointCloud();
    write3(d + "/out_vpoints.f32", vp->points_);
    write3(d + "/out_vcolors.f32", vp->colors_);
    auto vg = vol.ExtractVoxelGrid();
    const auto keys = vg->voxels_keys_.to_host();
    write_file(d + "/out_vg_keys.i32", keys.data(), keys.size() * 12);
    write3(d + "/out_vg_colors.f32", vg->voxels_colors_);
    const float org[4] = {vg->origin_[0], vg->origin_[1], vg->origin_[2], vg->voxel_size_};
    write_file(d + "/out_vg_origin.f32", org, 16);
    for (int valid = 0; valid < 2; ++valid) {
        auto rc = vol.Raycast(K, E[0], prm[9], valid == 1);
        const std::string s = valid ? "valid" : "all";
        write3(d + "/out_ray_" + s + "_points.f32", rc->points_);
        write3(d + "/out_ray_" + s + "_normals.f32", rc->normals_);
        write3(d + "/out_ray_" + s + "_colors.f32", rc->colors_);
    }
    vol.Reset();
    EXPECT(vol.ExtractPointCloud()->points_.size() == 0 && vol.ExtractVoxelGrid()->voxels_keys_.size() == 0);
    return fails ? 1 : 0;
}
