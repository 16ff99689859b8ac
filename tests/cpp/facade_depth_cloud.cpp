// PointCloud::CreateFromDepthImage / CreateFromRGBDImage through the header-compatible facade.  Without arguments: a
// compile-and-link check.  With DIR: the argument errors, then from DIR/params.f32 = {w, h, fx, fy, cx, cy, extrinsic
// row-major [16]}, DIR/depth.u16 [h][w] and DIR/color.u8 [h][w][3]:
//   out_d_points    CreateFromDepthImage(depth, K, E, 1000, 4, stride 3)
//   out_v_*         CreateFromRGBDImage(CreateFromColorAndDepth(color, depth, 1000, 4, false), K, E, true, 2.0, true)
//   out_a_*         the same with project_valid_depth_only = false and no normals
// Exit code 0 = all expectations met.
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/camera/pinhole_camera_intrinsic.h"
#include "cupoch/geometry/pointcloud.h"
#include "cupoch/geometry/rgbdimage.h"
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
    const auto prm = read_file<float>(d + "/params.f32");
    const int w = (int)prm[0], h = (int)prm[1];
    const camera::PinholeCameraIntrinsic K(w, h, prm[2], prm[3], prm[4], prm[5]);
    const Eigen::Matrix4f E = utility::from_row_major(prm.data() + 6);
    const auto depth = read_file<uint16_t>(d + "/depth.u16");
    const auto color = read_file<uint8_t>(d + "/color.u8");
    const geometry::Image di = image(depth.data(), w, h, 1, 2), ci = image(color.data(), w, h, 3, 1);
    {  // argument errors
        EXPECT(throws([&] { geometry::PointCloud::CreateFromDepthImage(di, K, E, 1000.f, 4.f, 0); }));
        EXPECT(throws([&] { geometry::PointCloud::CreateFromDepthImage(ci, K); }));
        EXPECT(throws([&] { geometry::PointCloud::CreateFromDepthImage(di, K, Eigen::Matrix4f()); }));  // singular
        geometry::RGBDImage raw(ci, di);  // uint16 depth: not an RGBDImage's float32 depth
        EXPECT(throws([&] { geometry::PointCloud::CreateFromRGBDImage(raw, K); }));
    }
    auto pd = geometry::PointCloud::CreateFromDepthImage(di, K, E, 1000.f, 4.f, 3);
    EXPECT(pd->HasPoints() && !pd->HasNormals() && !pd->HasColors());
    write3(d + "/out_d_points.f32", pd->points_);
    auto im = geometry::RGBDImage::CreateFromColorAndDepth(ci, di, 1000.f, 4.f, false);
    auto pv = geometry::PointCloud::CreateFromRGBDImage(*im, K, E, true, 2.0f, true);
    EXPECT(pv->HasNormals() && pv->HasColors() && pv->points_.size() < (size_t)w * h);
    write3(d + "/out_v_points.f32", pv->points_);
    write3(d + "/out_v_normals.f32", pv->normals_);
    write3(d + "/out_v_colors.f32", pv->colors_);
    auto pa = geometry::PointCloud::CreateFromRGBDImage(*im, K, E, false, 2.0f, false);
    EXPECT(pa->points_.size() == (size_t)w * h && pa->normals_.size() == 0);
    write3(d + "/out_a_points.f32", pa->points_);
    write3(d + "/out_a_colors.f32", pa->colors_);
    return fails ? 1 : 0;
}
