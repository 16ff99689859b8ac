// Bounding boxes and point-cloud cleanup through the header-compatible facade (cupoch/geometry/boundingvolume.h):
//   - the known answer of the reference's GetOrientedBoundingBox test (the 3 x 2 x 1 box: R = I, centre and extent
//     exact) and the argument rules (axis_no 3 and every_k_points 0 give empty clouds, an empty box still crops);
//   - with DIR: on DIR/points.f32 (with DIR/normals.f32) every call's output written to DIR/<name>.f32 for comparison
//     with the oracle: crop_aabb, crop_obb, pass_through, uniform, finite (points), obb (centre, R row-major, extent),
//     normalized, oriented (normals).
// Exit code 0 = all expectations met.
#include <cstdio>
#include <string>
#include <vector>

#include "cupoch/geometry/boundingvolume.h"
#include "cupoch/geometry/pointcloud.h"
#include "facade_check.h"

using namespace cupoch;

static void write_rows(const std::string &path, const std::vector<Eigen::Vector3f> &rows) {
    const std::vector<float> f = rows3(rows);
    write_file(path, f.data(), f.size() * sizeof(float));
}

int main(int argc, char **argv) {
    {
        std::vector<Eigen::Vector3f> pts;
        for (int x : {0, 3})
            for (int y : {0, 2})
                for (int z : {0, 1}) pts.push_back(Eigen::Vector3f((float)x, (float)y, (float)z));
        geometry::PointCloud pcd(pts);
        const geometry::OrientedBoundingBox obb = pcd.GetOrientedBoundingBox();
        EXPECT(obb.center_(0) == 1.5f && obb.center_(1) == 1.f && obb.center_(2) == 0.5f);
        EXPECT(obb.extent_(0) == 3.f && obb.extent_(1) == 2.f && obb.extent_(2) == 1.f);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) EXPECT(obb.R_(r, c) == (r == c ? 1.f : 0.f));
        EXPECT(obb.Volume() == 6.f && !obb.IsEmpty());
        const geometry::AxisAlignedBoundingBox<3> aabb = pcd.GetAxisAlignedBoundingBox();
        EXPECT(aabb.GetMaxExtent() == 3.f && aabb.Volume() == 6.f && aabb.GetCenter()(0) == 1.5f);
        EXPECT(pcd.Crop(obb)->GetPoints().size() == 8 && pcd.Crop(aabb)->GetPoints().size() == 8);
        EXPECT(pcd.PassThroughFilter(3, 0.f, 1.f)->IsEmpty());
        EXPECT(pcd.PassThroughFilter(0, 1.f, 5.f)->GetPoints().size() == 4);
        EXPECT(pcd.UniformDownSample(0)->IsEmpty());
        EXPECT(pcd.UniformDownSample(3)->GetPoints().size() == 2);
        const geometry::AxisAlignedBoundingBox<3> flat(Eigen::Vector3f(0, 0, 0), Eigen::Vector3f(3, 2, 0));
        EXPECT(flat.IsEmpty() && pcd.Crop(flat)->GetPoints().size() == 4);  // logged, and still cropped
        EXPECT(!pcd.OrientNormalsToAlignWithDirection());
        geometry::PointCloud empty;
        EXPECT(empty.GetOrientedBoundingBox().Volume() == 0.f && empty.RemoveNoneFinitePoints().IsEmpty());
    }
    if (argc == 2) {
        const std::string dir = argv[1];
        geometry::PointCloud pcd(rows3(read_file<float>(dir + "/points.f32")));
        pcd.SetNormals(rows3(read_file<float>(dir + "/normals.f32")));
        if (pcd.IsEmpty() || !pcd.HasNormals()) return 2;
        const geometry::AxisAlignedBoundingBox<3> box(Eigen::Vector3f(0.5f, 1.f, 0.25f), Eigen::Vector3f(2.f, 4.f, 0.75f));
        Eigen::Matrix3f R = Eigen::Matrix3f::Identity();
        R(0, 0) = 0.8660254f; R(0, 1) = -0.5f; R(1, 0) = 0.5f; R(1, 1) = 0.8660254f;
        const geometry::OrientedBoundingBox obox(Eigen::Vector3f(2.f, 2.f, 0.5f), R, Eigen::Vector3f(2.6f, 2.6f, 1.2f));
        write_rows(dir + "/crop_aabb.f32", pcd.Crop(box)->GetPoints());
        write_rows(dir + "/crop_obb.f32", pcd.Crop(obox)->GetPoints());
        write_rows(dir + "/pass_through.f32", pcd.PassThroughFilter(1, 0.25f, 0.75f)->GetPoints());
        write_rows(dir + "/uniform.f32", pcd.UniformDownSample(5)->GetPoints());
        const geometry::OrientedBoundingBox obb = pcd.GetOrientedBoundingBox();
        std::vector<float> o = {obb.center_(0), obb.center_(1), obb.center_(2)};
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) o.push_back(obb.R_(r, c));
        o.insert(o.end(), {obb.extent_(0), obb.extent_(1), obb.extent_(2)});
        write_file(dir + "/obb.f32", o.data(), o.size() * sizeof(float));
        geometry::PointCloud n1 = pcd;
        write_rows(dir + "/normalized.f32", n1.NormalizeNormals().GetNormals());
        geometry::PointCloud n2 = pcd;
        EXPECT(n2.OrientNormalsToAlignWithDirection(Eigen::Vector3f(0.f, 0.5f, 2.f)));
        write_rows(dir + "/oriented.f32", n2.GetNormals());
        write_rows(dir + "/finite.f32", pcd.RemoveNoneFinitePoints().GetPoints());
        EXPECT(pcd.HasNormals());
    }
    if (fails) return 1;
    std::printf("facade bounding boxes and cleanup: all expectations met\n");
    return 0;
}
