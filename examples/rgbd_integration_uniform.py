"""RGB-D integration into a uniform TSDF volume (the counterpart of the reference's advanced/rgbd_integration_uniform.py),
closed into the tracking step of KinectFusion: synthetic frames of three spheres seen from cameras on a ring are fused,
the surface is extracted and raycast from one view, and a moved copy of that view's surface is registered against the
raycast by point-to-plane ICP.  Depth maps are rendered analytically; there is no visualiser and no IO."""
import numpy as np

import cupoch_b200 as cph
from cupoch_b200.testing.datagen import gt_transform, ring_cameras, sphere_depth

W, H, VIEWS = 320, 240, 12
CENTRES, RADII = np.float32([[0, 0, 0], [0.45, 0.1, -0.2], [-0.2, 0.5, 0.25]]), (0.35, 0.2, 0.15)


def depth_map(K, E):
    """camera-z depth of the nearest sphere per pixel, 0 where every ray misses"""
    out = np.zeros((H, W), np.float32)
    for c, r in zip(CENTRES, RADII):
        Ec = E.copy()
        Ec[:3, 3] = E[:3, :3] @ c + E[:3, 3]
        d = sphere_depth(K, Ec, W, H, r)
        out = np.where((d > 0) & ((out == 0) | (d < out)), d, out)
    return out


def main():
    cams = ring_cameras(VIEWS, W, H)
    K = cams[0][0]
    intrinsic = cph.camera.PinholeCameraIntrinsic(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    volume = cph.integration.UniformTSDFVolume(length=2.0, resolution=256, sdf_trunc=0.04,
                                               color_type=cph.integration.TSDFVolumeColorType.RGB8)
    rng = np.random.default_rng(0)
    for _, E in cams:
        depth = cph.geometry.Image(np.round(depth_map(K, E) * 1000).astype(np.uint16))  # millimetres, as a sensor gives
        color = cph.geometry.Image(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        rgbd = cph.geometry.RGBDImage.create_from_color_and_depth(color, depth, depth_trunc=4.0, convert_rgb_to_intensity=False)
        volume.integrate(rgbd, intrinsic, E)
    print("extract_point_cloud:", len(volume.extract_point_cloud()), "points with normals")
    print("extract_voxel_point_cloud:", len(volume.extract_voxel_point_cloud()), "voxels in the band")
    print("extract_voxel_grid:", len(volume.extract_voxel_grid()), "voxels")
    mesh = volume.extract_triangle_mesh()
    mesh.compute_vertex_normals()
    print("extract_triangle_mesh:", len(mesh.vertices) if mesh.has_vertices() else 0, "vertices,",
          len(mesh.triangles) if mesh.has_triangles() else 0, "triangles, with vertex normals")

    E = cams[0][1]
    target = volume.raycast(intrinsic, E, 0.04)
    print("raycast:", len(target), "surface points predicted for view 0")
    # the source: view 0's surface back-projected, moved by the inverse of a known motion
    d = depth_map(K, E)
    v, u = np.nonzero(d > 0)
    cam = (np.stack([u, v, np.ones_like(u)], 1) @ np.linalg.inv(K.astype(np.float64)).T) * d[v, u, None]
    world = (cam - E[:3, 3]) @ E[:3, :3].astype(np.float64)
    T = gt_transform((1.0, -1.5, 2.0), (0.02, -0.01, 0.015))
    source = cph.geometry.PointCloud(((world - T[:3, 3]) @ T[:3, :3]).astype(np.float32))
    R = cph.registration
    res = R.registration_icp(source, target, 0.05, np.eye(4), R.TransformationEstimationPointToPlane(),
                             R.ICPConvergenceCriteria(1e-9, 1e-9, 60))
    print("point-to-plane ICP against the raycast: fitness %.3f, translation error %.2e m"
          % (res.fitness, np.linalg.norm(res.transformation[:3, 3] - T[:3, 3])))


if __name__ == "__main__":
    main()
