"""Voxel carving (the counterpart of the reference's advanced/voxel_carving.py): a dense grid around an object is carved
by depth maps and by silhouettes seen from cameras on a ring, then merged with the voxelised surface.  A sphere takes
the mesh's place and its depth maps are rendered analytically; there is no visualiser and no IO."""
import numpy as np

import cupoch_b200 as cph

W, H, RADIUS, VIEWS = 160, 120, 0.8, 12


def ring_camera(i):
    a = 2 * np.pi * i / VIEWS
    eye = np.array([2.5 * np.cos(a), 2.5 * np.sin(a), 0.5 * np.sin(3 * a)])
    zc = -eye / np.linalg.norm(eye)
    xc = np.cross(zc, [0, 0, 1.0])
    xc /= np.linalg.norm(xc)
    R = np.stack([xc, np.cross(zc, xc), zc])
    E = np.eye(4)
    E[:3, :3], E[:3, 3] = R, -R @ eye
    intr = cph.camera.PinholeCameraIntrinsic(W, H, 0.9 * W, 0.9 * W, (W - 1) / 2, (H - 1) / 2)
    return cph.camera.PinholeCameraParameters(intr, E)


def depth_map(cam):
    """camera-z depth of the sphere per pixel, 0 where the ray misses"""
    K, E = cam.intrinsic.intrinsic_matrix.astype(np.float64), cam.extrinsic.astype(np.float64)
    uu, vv = np.meshgrid(np.arange(W), np.arange(H))
    rays = np.stack([uu, vv, np.ones_like(uu)], -1).reshape(-1, 3) @ np.linalg.inv(K).T
    c, d = -E[:3, :3].T @ E[:3, 3], rays @ E[:3, :3]
    a, b, cc = np.sum(d * d, 1), 2 * d @ c, c @ c - RADIUS ** 2
    disc = b * b - 4 * a * cc
    return np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0).reshape(H, W).astype(np.float32)


if __name__ == "__main__":
    voxel_size = 2.0 / 96
    carved_depth = cph.geometry.VoxelGrid.create_dense((-1, -1, -1), voxel_size, 2, 2, 2)
    carved_silhouette = cph.geometry.VoxelGrid.create_dense((-1, -1, -1), voxel_size, 2, 2, 2)
    print("dense grid:", len(carved_depth), "voxels")
    for i in range(VIEWS):
        cam = ring_camera(i)
        depth = depth_map(cam)
        carved_depth.carve_depth_map(cph.geometry.Image(depth), cam)
        # the reference applies the depth test (d > 0 and z >= d) to silhouettes too, so the mask is a float32 image
        # whose set pixels hold a value below every depth in front of the camera
        mask = np.where(depth > 0, np.float32(1e-3), np.float32(0))
        carved_silhouette.carve_silhouette(cph.geometry.Image(mask), cam)
    print("carved by %d depth maps: %d voxels; by %d silhouettes: %d voxels" % (VIEWS, len(carved_depth), VIEWS, len(carved_silhouette)))

    rng = np.random.default_rng(0)
    surface = rng.normal(size=(200_000, 3))
    surface = (RADIUS * surface / np.linalg.norm(surface, axis=1, keepdims=True)).astype(np.float32)
    voxel_surface = cph.geometry.VoxelGrid.create_from_point_cloud_within_bounds(cph.geometry.PointCloud(surface), voxel_size,
                                                                                (-1, -1, -1), (1, 1, 1))
    print("surface voxels:", len(voxel_surface))
    carved_depth += voxel_surface
    print("carved + surface:", len(carved_depth), "voxels")
    centres = (carved_depth.get_voxels()[0] + 0.5) * voxel_size - 1
    print("largest centre radius %.3f (sphere radius %.2f)" % (np.linalg.norm(centres, axis=1).max(), RADIUS))
