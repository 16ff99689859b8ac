"""geometry::DistanceTransform: the Euclidean distance field of a voxelised shape (the reference's
examples/python/robotics/distancetransform.py voxelises a mesh; here the VoxelGrid comes from a synthetic cloud on a
sphere, and examples/voxelize_mesh.py runs the mesh flow with VoxelGrid.create_from_triangle_mesh_within_bounds)."""
import numpy as np

import cupoch_b200 as cph

if __name__ == "__main__":
    cubic_size, voxel_resolution = 1.0, 128
    rng = np.random.default_rng(1)
    d = rng.standard_normal((200_000, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    sphere = (0.3 * d).astype(np.float32)
    target = cph.geometry.VoxelGrid.create_from_point_cloud_within_bounds(
        cph.geometry.PointCloud(sphere), voxel_size=cubic_size / voxel_resolution,
        min_bound=(-cubic_size / 2, -cubic_size / 2, -cubic_size / 2),
        max_bound=(cubic_size / 2, cubic_size / 2, cubic_size / 2))
    dt = cph.geometry.DistanceTransform(cubic_size / voxel_resolution, voxel_resolution)
    dt.compute_edt(target)
    print(dt, "from", len(target), "voxels")
    print("distance at the centre (about 0.3):", dt.get_distance((0.0, 0.0, 0.0)))
    q = rng.uniform(-0.5, 0.5, (1_000_000, 3)).astype(np.float32)
    dist = dt.get_distances(q).cpu()
    print("clearance of 1 M random points: mean %.4f, max %.4f" % (dist.mean(), dist.max()))
    found, voxel = dt.get_voxel((0.0, 0.0, 0.0))
    print("voxel at the centre:", found, voxel)
    field = dt.to_torch()  # zero-copy [128, 128, 128] float32 CUDA tensor
    print("cells within one voxel of the surface:", int((field <= cubic_size / voxel_resolution).sum()))
