"""collision::ComputeIntersection: a voxelised shape slid through a copy of itself (the reference's
examples/python/robotics/collision_voxelgrid.py without the visualiser; the reference voxelises a mesh, here the
VoxelGrid comes from a synthetic cloud on a sphere (examples/voxelize_mesh.py voxelises a mesh), and the query is moved by assigning its origin because there is no
VoxelGrid::Translate in this engine).  Then a box, a sphere and a capsule against the same grid."""
import numpy as np

import cupoch_b200 as cph

if __name__ == "__main__":
    cubic_size, voxel_resolution = 1.0, 128.0
    rng = np.random.default_rng(1)
    d = rng.standard_normal((200_000, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    target = cph.geometry.VoxelGrid.create_from_point_cloud_within_bounds(
        cph.geometry.PointCloud((0.2 * d).astype(np.float32)), voxel_size=cubic_size / voxel_resolution,
        min_bound=(-cubic_size / 2, -cubic_size / 2, -cubic_size / 2),
        max_bound=(cubic_size / 2, cubic_size / 2, cubic_size / 2))
    query = cph.geometry.VoxelGrid()
    query.voxel_size, query.voxels_keys = target.voxel_size, target.voxels_keys
    query.origin = target.origin + np.array([-0.45, 0.0, 0.0], np.float32)

    dh = 0.06
    for i in range(15):
        query.origin = query.origin + np.array([dh, 0.0, 0.0], np.float32)
        ans = cph.collision.compute_intersection(target, query, 0.0)
        print(i, ans, "target voxels hit:", len(np.unique(ans.get_first_collision_indices())),
              "query voxels hit:", len(np.unique(ans.get_second_collision_indices())))

    prims = cph.collision.PrimitiveArray()
    prims.append(cph.collision.Box([0.1, 0.1, 0.1], np.array([[1, 0, 0, 0.2], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])))
    prims.append(cph.collision.Sphere(0.05, (0.0, 0.0, 0.0)))  # inside the hollow sphere: no collision
    prims.append(cph.collision.Capsule(0.02, 0.6))              # along z through the centre: hits both poles
    ans = cph.collision.compute_intersection(target, prims, 0.0)
    print(ans, "primitives that collide:", ans.get_second_collision_indices().tolist())
