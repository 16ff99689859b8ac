#!/usr/bin/env python3
"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / synccheck):
   compute-sanitizer --tool memcheck python tools/sanitize_small.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cupoch_b200 as cph
from cupoch_b200.testing import datagen

R, G = cph.registration, cph.geometry
n = int(os.environ.get('SANITIZE_POINTS', '20000'))   # >= 8192 points: the certified regime runs with helper blocks
tgt, tn = datagen.surface(n, 11)
tc = datagen.texture(tgt)
src, sn, sc = datagen.make_source(tgt, datagen.gt_transform((-1, 1.5, 2), (0.01, -0.005, 0.008)), 13, 14, 5e-4,
                                  attrs=[(tn, True), (tc, False)])
s, t = G.PointCloud(src), G.PointCloud(tgt)
s.normals, s.colors, t.normals, t.colors = sn, sc, tn, tc
crit = R.ICPConvergenceCriteria(0, 0, 12)         # 13 launches: searching regime, then the certified one (DMMA, cp.async pipeline, fused tail)
for name, fn in (("p2p", lambda: R.registration_icp(s, t, 0.03, np.eye(4), R.TransformationEstimationPointToPoint(), crit)),
                 ("p2plane", lambda: R.registration_icp(s, t, 0.03, np.eye(4), R.TransformationEstimationPointToPlane(), crit)),
                 ("symmetric", lambda: R.registration_icp(s, t, 0.03, np.eye(4), R.TransformationEstimationSymmetricMethod(), crit)),
                 ("gicp", lambda: R.registration_generalized_icp(s, t, 0.03, np.eye(4), None, crit)),
                 ("colored", lambda: R.registration_colored_icp(s, t, 0.03, np.eye(4), crit))):
    r = fn()
    print(name, "fitness %.3f" % r.fitness, "corr", len(r.correspondence_set))
tree = G.KDTreeFlann(t)
print("knn", tree.search_knn(s.points, 8)[0], "radius", tree.search_radius(s.points, 0.01, 5)[0])
d = t.voxel_down_sample(0.05)
print("voxel", len(d))
t2 = G.PointCloud(tgt)
t2.estimate_normals(G.KDTreeSearchParamKNN(10))
print("normals ok", bool(np.isfinite(t2.normals.cpu()).all()))
t2.estimate_normals(G.KDTreeSearchParamRadius(0.03, 20))
print("normals (radius) ok", bool(np.isfinite(t2.normals.cpu()).all()))
og = G.OccupancyGrid(0.05, 96)
rng = np.random.default_rng(3)
scan = (rng.standard_normal((5000, 3)).astype(np.float32) * 1.2).astype(np.float32)
og.insert(scan, (0.1, 0.0, -0.1), 2.0)
og.add_voxels(rng.integers(0, 96, (500, 3)).astype(np.int32), True)
og.set_free_area((-0.5, -0.5, -0.5), (0.5, 0.5, 0.5))
print("occupancy grid known voxels", len(og.extract_known_voxels()[1]), "occupied", len(og.extract_occupied_voxels()[1]))
small = G.PointCloud(tgt[:4000])
small.normals = tn[:4000]
print("fpfh", R.compute_fpfh_feature(small, G.KDTreeSearchParamKNN(10)).cpu().shape, "dbscan clusters", int(small.cluster_dbscan(0.02, 5).cpu().max()) + 1)
out, idx = small.remove_radius_outlier(4, 0.02)
print("radius outlier kept", len(out), "gaussian", len(small.gaussian_filter(0.02, 1e-4, 20)))
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
vol = cph.integration.UniformTSDFVolume(2.0, 48, 0.08, cph.integration.TSDFVolumeColorType.RGB8)
for K, E in ring_cameras(3, 64, 48):
    d16 = (sphere_depth(K, E, 64, 48, 0.6) * 1000).astype(np.uint16)
    im = G.RGBDImage.create_from_color_and_depth(G.Image(np.full((48, 64, 3), 90, np.uint8)), G.Image(d16), convert_rgb_to_intensity=False)
    intr = cph.camera.PinholeCameraIntrinsic(64, 48, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    vol.integrate(im, intr, E)
print("tsdf points", len(vol.extract_point_cloud()), "voxels", len(vol.extract_voxel_grid()),
      "raycast", len(vol.raycast(intr, E, 0.08)), len(vol.raycast(intr, E, 0.08, False)))
mesh = vol.extract_triangle_mesh()
mesh.compute_vertex_normals()
print("tsdf mesh vertices", len(mesh.vertices), "triangles", len(mesh.triangles), "vertex normals", len(mesh.vertex_normals))
print("rgbd points", len(G.PointCloud.create_from_rgbd_image(im, intr, E, True, -1.0, True)),
      len(G.PointCloud.create_from_rgbd_image(im, intr, E, False, 2.4, True)),
      "depth points", len(G.PointCloud.create_from_depth_image(G.Image(d16), intr, E, 1000.0, 4.0, 3)))
mesh.compute_edge_list()
filtered = [mesh.filter_sharpen(2, 0.1), mesh.filter_smooth_simple(2, G.FilterScope.Color),
            mesh.filter_smooth_laplacian(2, 0.5, G.FilterScope.Vertex), mesh.filter_smooth_taubin(2)]
sampled = mesh.sample_points_uniformly(3000, True)
print("mesh edges", len(mesh.edge_list), "filtered", [len(m.vertices) for m in filtered], "area %.4f" % mesh.get_surface_area(),
      "sampled", len(sampled.points), len(sampled.normals), len(sampled.colors))
mesh_grid = G.VoxelGrid.create_from_triangle_mesh(mesh, 0.05)
print("mesh voxels", len(mesh_grid), "within bounds", len(G.VoxelGrid.create_from_triangle_mesh_within_bounds(mesh, 0.1, (-1, -1, -1), (0.2, 1, 1))))
soup = G.TriangleMesh(mesh.vertices.cpu()[mesh.triangles.cpu().reshape(-1)], np.arange(3 * len(mesh.triangles), dtype=np.int32).reshape(-1, 3))
both = mesh + soup
print("self-intersections", len(both.get_self_intersecting_triangles()), "soup", len(soup.get_self_intersecting_triangles()))
big = G.TriangleMesh(np.concatenate([mesh.vertices.cpu(), np.float32([[-2, -2, 0], [2, -2, 0.1], [0, 2, -0.1], [-2, 0, -1], [2, 0.2, 1], [0, -0.2, 1]])]),
                     np.concatenate([mesh.triangles.cpu(), len(mesh.vertices) + np.int32([[0, 1, 2], [3, 4, 5]])]).astype(np.int32))
print("large-tier self-intersections", len(big.get_self_intersecting_triangles()))
soup.remove_duplicated_vertices().remove_duplicated_triangles().remove_degenerate_triangles().remove_unreferenced_vertices()
print("welded soup", len(soup.vertices), len(soup.triangles))
