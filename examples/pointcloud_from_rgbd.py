"""A point cloud from an RGB-D frame (the counterpart of the reference's PointCloud.create_from_rgbd_image /
create_from_depth_image use in its examples), then two frames registered by point-to-plane ICP with no host round trip:
the clouds stay on the device from the depth image to registration_icp.  Depth maps of three spheres are rendered
analytically; there is no visualiser and no IO."""
import numpy as np

import cupoch_b200 as cph
from cupoch_b200.testing.datagen import gt_transform, ring_cameras, sphere_depth

W, H = 320, 240
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
    K, E1 = ring_cameras(8, W, H)[0]
    intrinsic = cph.camera.PinholeCameraIntrinsic(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    motion = gt_transform((1.0, -1.5, 2.0), (0.02, -0.01, 0.015)).astype(np.float32)
    E2 = motion @ E1  # the camera moved by `motion` in its own frame
    rng = np.random.default_rng(0)
    clouds = []
    for E in (E1, E2):
        depth = cph.geometry.Image(np.round(depth_map(K, E) * 1000).astype(np.uint16))  # millimetres, as a sensor gives
        color = cph.geometry.Image(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        rgbd = cph.geometry.RGBDImage.create_from_color_and_depth(color, depth, depth_trunc=4.0, convert_rgb_to_intensity=False)
        pc = cph.geometry.PointCloud.create_from_rgbd_image(rgbd, intrinsic, compute_normals=True)  # camera frame
        print("create_from_rgbd_image:", len(pc), "points with colours and structured normals")
        clouds.append(pc)
    coarse = cph.geometry.PointCloud.create_from_depth_image(depth, intrinsic, E2, stride=4)
    print("create_from_depth_image(stride=4):", len(coarse), "points in the world frame")

    target, source = clouds
    target.estimate_normals(cph.geometry.KDTreeSearchParamKNN(20))
    R = cph.registration
    res = R.registration_icp(source, target, 0.05, np.eye(4), R.TransformationEstimationPointToPlane(),
                             R.ICPConvergenceCriteria(1e-9, 1e-9, 60))
    want = np.linalg.inv(motion.astype(np.float64))  # camera 2 -> camera 1
    print("registration_icp: fitness %.3f, pose error %.2e" % (res.fitness, np.abs(np.asarray(res.transformation) - want).max()))


if __name__ == "__main__":
    main()
