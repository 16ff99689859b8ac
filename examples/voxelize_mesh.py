"""VoxelGrid.create_from_triangle_mesh_within_bounds: a mesh becomes a voxel grid, which then feeds the distance
transform and collision checks (the flow of the reference's examples/python/robotics/distancetransform.py and
collision_voxelgrid.py).  The mesh is extracted from a TSDF volume that fused eight synthetic views of a sphere."""
import numpy as np

import cupoch_b200 as cph
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth

if __name__ == "__main__":
    G = cph.geometry
    w, h = 320, 240
    vol = cph.integration.UniformTSDFVolume(2.0, 256, 0.04, cph.integration.TSDFVolumeColorType.NoColor)
    for K, E in ring_cameras(8, w, h):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((h, w, 3), np.uint8)), G.Image(d16), 1000.0, 100.0)
        vol.integrate(im, cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    mesh = vol.extract_triangle_mesh()
    print(mesh, "bounds", mesh.get_min_bound(), mesh.get_max_bound())

    cubic_size, voxel_resolution = 2.0, 128
    vs = cubic_size / voxel_resolution
    grid = G.VoxelGrid.create_from_triangle_mesh_within_bounds(mesh, vs, (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    print("mesh voxels:", len(grid), "around the mesh's own bounds:", len(G.VoxelGrid.create_from_triangle_mesh(mesh, vs)))

    dt = G.DistanceTransform(vs, voxel_resolution)
    dt.compute_edt(grid)
    print("distance at the centre (about 0.6):", dt.get_distance((0.0, 0.0, 0.0)))

    samples = mesh.sample_points_uniformly(200_000)
    points = G.VoxelGrid.create_from_point_cloud_within_bounds(samples, vs, (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    ans = cph.collision.compute_intersection(grid, points, 0.0)
    print("voxels of the mesh's samples:", len(points), "colliding with the mesh grid:",
          len(np.unique(ans.get_second_collision_indices())))
