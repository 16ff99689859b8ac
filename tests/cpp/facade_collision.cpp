// collision::ComputeIntersection through the header-compatible facade.  With DIR: the reference's TEST(Collision,
// VoxelVoxel) with the keys assigned to voxels_keys_, and the primitives' bounding boxes; then (DIR/params.f32 =
// {vs_a, ax, ay, az, vs_b, bx, by, bz, margin, occ_vs, occ_res}, DIR/keys_a.i32, DIR/keys_b.i32, DIR/prims.f32 = per
// primitive {type, transform row-major [16], lengths [3], radius, height}, DIR/occ_cells.i32): the pairs of A x B,
// A x prims, prims x A, occ x B and B x occ are written to DIR/out_{ab,ap,pa,ob,bo}.i32.
// Exit code 0 = all expectations met.
#include <cstdio>
#include <string>
#include <vector>

#include "cupoch/collision/collision.h"
#include "cupoch/collision/primitives.h"
#include "cupoch/geometry/occupancygrid.h"
#include "cupoch/geometry/voxelgrid.h"
#include "facade_check.h"

using namespace cupoch;

static std::vector<Eigen::Vector3i> keys3(const std::vector<int32_t> &flat) {
    std::vector<Eigen::Vector3i> k;
    for (size_t i = 0; i + 2 < flat.size(); i += 3) k.push_back(Eigen::Vector3i(flat[i], flat[i + 1], flat[i + 2]));
    return k;
}

static void write_pairs(const std::string &path, const collision::CollisionResult &r) {
    std::vector<int32_t> flat;
    for (const auto &p : r.GetCollisionIndexPairs()) flat.insert(flat.end(), {p[0], p[1]});
    write_file(path, flat.data(), flat.size() * sizeof(int32_t));
}

static Eigen::Matrix4f row_major(const float *m) { return utility::from_row_major(m); }

int main(int argc, char **argv) {
    if (argc != 2) return 0;  // compile-and-link check only
    {  // TEST(Collision, VoxelVoxel)
        geometry::VoxelGrid v1, v2;
        EXPECT(!collision::ComputeIntersection(v1, v2)->IsCollided());
        v1.voxel_size_ = v2.voxel_size_ = 1.0f;
        v1.voxels_keys_ = std::vector<Eigen::Vector3i>{Eigen::Vector3i(0, 0, 0)};
        v2.voxels_keys_ = std::vector<Eigen::Vector3i>{Eigen::Vector3i(0, 0, 0)};
        EXPECT(collision::ComputeIntersection(v1, v2)->IsCollided());
        v1.voxels_keys_ = std::vector<Eigen::Vector3i>{Eigen::Vector3i(0, 0, 0), Eigen::Vector3i(5, 0, 0)};
        v2.voxels_keys_ = std::vector<Eigen::Vector3i>{Eigen::Vector3i(0, 0, 0), Eigen::Vector3i(10, 0, 0)};
        auto r = collision::ComputeIntersection(v1, v2);
        EXPECT(r->collision_index_pairs_.size() == 1);
        EXPECT(r->GetCollisionIndexPairs()[0][0] == 0 && r->GetCollisionIndexPairs()[0][1] == 0);
        EXPECT(r->first_ == collision::CollisionResult::CollisionType::VoxelGrid);
        EXPECT(r->GetFirstCollisionIndices() == std::vector<size_t>{0} && r->GetSecondCollisionIndices() == std::vector<size_t>{0});
        v1.voxel_size_ = 0.0f;  // rejected: logged, empty result
        EXPECT(!collision::ComputeIntersection(v1, v2)->IsCollided());
    }
    {  // bounding boxes (primitives.h as written)
        collision::Sphere s(2.0f, Eigen::Vector3f(1.f, 2.f, 3.f));
        const auto b = s.GetAxisAlignedBoundingBox();
        EXPECT(b.GetMinBound()[0] == -1.f && b.GetMaxBound()[2] == 5.f);
        collision::Box box(Eigen::Vector3f(2.f, 4.f, 6.f));
        EXPECT(box.GetAxisAlignedBoundingBox().GetMaxBound()[1] == 2.f);
        collision::Capsule c(0.5f, 2.f);
        EXPECT(c.GetAxisAlignedBoundingBox().GetMaxBound()[2] == 1.5f && c.GetAxisAlignedBoundingBox().GetMinBound()[0] == -0.5f);
    }
    const std::string dir = argv[1];
    const std::vector<float> prm = read_file<float>(dir + "/params.f32");
    if (prm.size() != 11) return 2;
    geometry::VoxelGrid A, B;
    A.voxel_size_ = prm[0];
    A.origin_ = Eigen::Vector3f(prm[1], prm[2], prm[3]);
    A.voxels_keys_ = keys3(read_file<int32_t>(dir + "/keys_a.i32"));
    B.voxel_size_ = prm[4];
    B.origin_ = Eigen::Vector3f(prm[5], prm[6], prm[7]);
    B.voxels_keys_ = keys3(read_file<int32_t>(dir + "/keys_b.i32"));
    const float margin = prm[8];
    collision::PrimitiveArray prims;
    const std::vector<float> pf = read_file<float>(dir + "/prims.f32");
    for (size_t i = 0; i + 21 < pf.size(); i += 22) {
        const int type = (int)pf[i];
        const Eigen::Matrix4f T = row_major(&pf[i + 1]);
        const float *l = &pf[i + 17], r = pf[i + 20], h = pf[i + 21];
        if (type == 1) prims.push_back(collision::Box(Eigen::Vector3f(l[0], l[1], l[2]), T));
        else if (type == 2) {
            collision::Sphere s(r);
            s.transform_ = T;
            prims.push_back(s);
        } else if (type == 3) prims.push_back(collision::Capsule(r, h, T));
        else prims.push_back(collision::Cylinder(r, h, T));
    }
    geometry::OccupancyGrid occ(prm[9], (size_t)prm[10]);
    occ.AddVoxels(utility::device_vector<Eigen::Vector3i>(keys3(read_file<int32_t>(dir + "/occ_cells.i32"))), true);

    write_pairs(dir + "/out_ab.i32", *collision::ComputeIntersection(A, B, margin));
    write_pairs(dir + "/out_ap.i32", *collision::ComputeIntersection(A, prims, margin));
    write_pairs(dir + "/out_pa.i32", *collision::ComputeIntersection(prims, A, margin));
    write_pairs(dir + "/out_ob.i32", *collision::ComputeIntersection(occ, B, margin));
    write_pairs(dir + "/out_bo.i32", *collision::ComputeIntersection(B, occ, margin));
    if (fails) return 1;
    std::printf("facade collision: all expectations met\n");
    return 0;
}
