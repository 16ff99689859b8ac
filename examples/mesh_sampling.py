"""Mesh sampling (the counterpart of the reference's basic/mesh_sampling.py): a sphere fused from synthetic depth frames
is extracted as a mesh and turned back into point clouds by sample_points_uniformly, with interpolated vertex normals
and colours, or with the triangles' normals.  A second sample, moved by a known motion, is then registered to the first
by point-to-plane ICP: model-to-scan registration against a fused model.  The reference example uses meshes.knot() and
a viewer; there is no visualiser and no IO here."""
import numpy as np

import cupoch_b200 as cph
from cupoch_b200.testing.datagen import gt_transform, ring_cameras, sphere_depth

W, H = 320, 240


def sphere_mesh():
    cams = ring_cameras(8, W, H)
    K = cams[0][0]
    intrinsic = cph.camera.PinholeCameraIntrinsic(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    volume = cph.integration.UniformTSDFVolume(2.0, 192, 0.04, cph.integration.TSDFVolumeColorType.RGB8)
    rng = np.random.default_rng(1)
    for _, E in cams:
        depth = cph.geometry.Image(np.round(sphere_depth(K, E, W, H, 0.6) * 1000).astype(np.uint16))
        color = cph.geometry.Image(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        volume.integrate(cph.geometry.RGBDImage.create_from_color_and_depth(color, depth, depth_trunc=4.0,
                                                                            convert_rgb_to_intensity=False), intrinsic, E)
    mesh = volume.extract_triangle_mesh()
    mesh.compute_vertex_normals()
    return mesh


def main():
    mesh = sphere_mesh()
    print("mesh:", len(mesh.vertices), "vertices,", len(mesh.triangles), "triangles, area %.4f" % mesh.get_surface_area())
    pcd = mesh.sample_points_uniformly(number_of_points=500)
    print("sample_points_uniformly(500):", len(pcd.points), "points, normals", pcd.has_normals(), "colours", pcd.has_colors())
    pcd = mesh.sample_points_uniformly(number_of_points=200000, use_triangle_normal=True)
    print("with triangle normals:", len(pcd.normals), "normals; the mesh now has triangle normals:", mesh.has_triangle_normals())

    model = mesh.sample_points_uniformly(100000)
    scan = cph.geometry.PointCloud(mesh.sample_points_uniformly(200000).points.cpu()[1::2])
    T = gt_transform((2.0, -1.0, 1.5), (0.02, -0.01, 0.015))
    scan.transform(T)
    scan.estimate_normals(cph.geometry.KDTreeSearchParamKNN(20))
    R = cph.registration
    res = R.registration_icp(model, scan, 0.1, np.eye(4), R.TransformationEstimationPointToPlane(),
                             R.ICPConvergenceCriteria(1e-8, 1e-8, 60))
    print("registration_icp: fitness %.4f, largest pose error %.2e" % (res.fitness, np.abs(res.transformation - T).max()))


if __name__ == "__main__":
    main()
