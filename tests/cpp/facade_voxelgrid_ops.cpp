// The VoxelGrid operations through the header-compatible facade.  Without arguments: a compile-and-link check.  With
// DIR: known answers (a 2x3x4 CreateDense, GetVoxelCenterCoordinate's zero vector, the camera accessors, the argument
// errors), then from DIR/params.f32 = {vs, ox, oy, oz, occ_vs, occ_res, w, h, fx, fy, cx, cy, extrinsic row-major [16]},
// DIR/{keys_a, keys_b, occ_cells}.i32, DIR/{colors_a, colors_b, queries, depth}.f32 and DIR/idx.i64 the results of
// CheckIfIncluded, +=, AddVoxels, SelectByIndex (both), PaintIndexedColor, CarveDepthMap of a dense grid and both
// CreateFromOccupancyGrid calls are written to DIR/out_*.  Exit code 0 = all expectations met.
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "cupoch/camera/pinhole_camera_intrinsic.h"
#include "cupoch/camera/pinhole_camera_parameters.h"
#include "cupoch/geometry/image.h"
#include "cupoch/geometry/occupancygrid.h"
#include "cupoch/geometry/voxelgrid.h"
#include "facade_check.h"

using namespace cupoch;

static std::vector<Eigen::Vector3i> keys3(const std::vector<int32_t> &flat) {
    std::vector<Eigen::Vector3i> k;
    for (size_t i = 0; i + 2 < flat.size(); i += 3) k.push_back(Eigen::Vector3i(flat[i], flat[i + 1], flat[i + 2]));
    return k;
}
static geometry::VoxelGrid grid(const std::string &d, const char *name, float vs, const Eigen::Vector3f &o) {
    geometry::VoxelGrid g;
    g.voxel_size_ = vs;
    g.origin_ = o;
    g.voxels_keys_ = keys3(read_file<int32_t>(d + "/keys_" + name + ".i32"));
    g.voxels_colors_ = rows3(read_file<float>(d + "/colors_" + name + ".f32"));
    return g;
}
static void write_grid(const std::string &d, const std::string &name, const geometry::VoxelGrid &g) {
    const auto k = g.voxels_keys_.to_host();
    const auto c = g.voxels_colors_.to_host();
    write_file(d + "/out_" + name + "_keys.i32", k.data(), k.size() * 12);
    write_file(d + "/out_" + name + "_colors.f32", c.data(), c.size() * 12);
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
    {  // known answers
        auto g = geometry::VoxelGrid::CreateDense(Eigen::Vector3f(0.f, 0.f, 0.f), 0.5f, 1.f, 1.5f, 2.f);
        const auto k = g->voxels_keys_.to_host();
        EXPECT(k.size() == 24 && k[0][2] == 0 && k[1][2] == 1 && k[4][1] == 1 && k[23][0] == 1 && k[23][1] == 2 && k[23][2] == 3);
        EXPECT(g->GetVoxelCenterCoordinate(Eigen::Vector3i(1, 2, 3))[2] == 1.75f);
        EXPECT(g->GetVoxelCenterCoordinate(Eigen::Vector3i(5, 0, 0))[0] == 0.f);
        const auto bp = g->GetVoxelBoundingPoints(Eigen::Vector3i(0, 0, 0));
        EXPECT(bp[0][0] == 0.f && bp[7][0] == 0.5f && bp[1][2] == 0.5f && bp[2][0] == 0.5f && bp[4][1] == 0.5f);
        const auto inc = g->CheckIfIncluded({Eigen::Vector3f(0.1f, 0.1f, 0.1f), Eigen::Vector3f(-0.1f, 0.f, 0.f),
                                             Eigen::Vector3f(std::nanf(""), 0.f, 0.f)});
        EXPECT(inc[0] && !inc[1] && !inc[2]);
        EXPECT(throws([] { geometry::VoxelGrid::CreateDense(Eigen::Vector3f(0.f, 0.f, 0.f), 0.f, 1.f, 1.f, 1.f); }));
        EXPECT(throws([&] { g->SelectByIndex(utility::device_vector<size_t>(std::vector<size_t>{24})); }));
        geometry::VoxelGrid other = *g;
        other.origin_ = Eigen::Vector3f(1.f, 0.f, 0.f);
        EXPECT(throws([&] { *g += other; }));
        g->AddVoxel(geometry::Voxel(Eigen::Vector3i(0, 0, 0), Eigen::Vector3f(0.f, 0.f, 0.f)));
        EXPECT(g->voxels_keys_.size() == 24 && g->voxels_colors_.to_host()[0][0] == 1.f);  // the existing voxel stays
        camera::PinholeCameraIntrinsic intr(64, 48, 50.f, 51.f, 31.5f, 23.5f);
        EXPECT(intr.IsValid() && intr.GetFocalLength().second == 51.f && intr.GetPrincipalPoint().first == 31.5f);
        EXPECT(!camera::PinholeCameraIntrinsic().IsValid());
        camera::PinholeCameraParameters cam;
        cam.intrinsic_ = intr;
        geometry::Image wrong;
        wrong.Prepare(63, 48, 1, 4);
        EXPECT(throws([&] { g->CarveDepthMap(wrong, cam); }));
    }
    const auto p = read_file<float>(d + "/params.f32");
    if (p.size() != 28) return 3;
    const float vs = p[0];
    const Eigen::Vector3f o(p[1], p[2], p[3]);
    auto a = grid(d, "a", vs, o), b = grid(d, "b", vs, o);
    const auto q = rows3(read_file<float>(d + "/queries.f32"));
    const auto inc = a.CheckIfIncluded(q);
    std::vector<uint8_t> inc8(inc.begin(), inc.end());
    write_file(d + "/out_included.u8", inc8.data(), inc8.size());
    write_grid(d, "merge", a + b);
    {
        geometry::VoxelGrid c = a;
        const auto kb = b.voxels_keys_.to_host();
        const auto cb = b.voxels_colors_.to_host();
        std::vector<geometry::Voxel> vox;
        for (size_t i = 0; i < kb.size(); ++i) vox.push_back(geometry::Voxel(kb[i], cb[i]));
        c.AddVoxels(vox);
        write_grid(d, "add", c);
    }
    const auto idx64 = read_file<int64_t>(d + "/idx.i64");
    const utility::device_vector<size_t> idx(std::vector<size_t>(idx64.begin(), idx64.end()));
    write_grid(d, "select", *a.SelectByIndex(idx));
    write_grid(d, "invert", *a.SelectByIndex(idx, true));
    {
        geometry::VoxelGrid c = a;
        c.PaintIndexedColor(idx, Eigen::Vector3f(0.25f, 0.5f, 0.75f));
        write_grid(d, "paint", c);
    }
    {
        const int w = (int)p[6], h = (int)p[7];
        camera::PinholeCameraParameters cam;
        cam.intrinsic_ = camera::PinholeCameraIntrinsic(w, h, p[8], p[9], p[10], p[11]);
        cam.extrinsic_ = utility::from_row_major(&p[12]);
        const auto depth = read_file<float>(d + "/depth.f32");
        geometry::Image img;
        img.Prepare(w, h, 1, 4);
        img.data_ = std::vector<uint8_t>(reinterpret_cast<const uint8_t *>(depth.data()),
                                         reinterpret_cast<const uint8_t *>(depth.data()) + depth.size() * 4);
        auto g = geometry::VoxelGrid::CreateDense(Eigen::Vector3f(-1.f, -1.f, -1.f), 2.f / 64, 2.f, 2.f, 2.f);
        g->CarveDepthMap(img, cam);
        write_grid(d, "carve", *g);
    }
    {
        geometry::OccupancyGrid occ(p[4], (size_t)p[5]);
        utility::device_vector<Eigen::Vector3i> cells(keys3(read_file<int32_t>(d + "/occ_cells.i32")));
        occ.AddVoxels(cells, true);
        auto v = geometry::VoxelGrid::CreateFromOccupancyGrid(occ);
        write_grid(d, "occvg", *v);
        const float vo[3] = {v->origin_[0], v->origin_[1], v->origin_[2]};
        write_file(d + "/out_occvg_origin.f32", vo, 12);
        auto pc = geometry::PointCloud::CreateFromOccupancyGrid(occ);
        const auto pts = pc->points_.to_host();
        const auto cols = pc->colors_.to_host();
        write_file(d + "/out_occpc_points.f32", pts.data(), pts.size() * 12);
        write_file(d + "/out_occpc_colors.f32", cols.data(), cols.size() * 12);
    }
    return fails ? 1 : 0;
}
