"""RGB-D integration into a scalable TSDF volume (the counterpart of the reference's advanced/rgbd_integration.py):
synthetic frames of three spheres seen from cameras on a ring are fused into 16^3-voxel units allocated only near the
surfaces, then the surface is extracted.  The allocated units' device bytes are printed next to those of a dense
UniformTSDFVolume of the same voxel length over the same box.  Depth maps are rendered analytically; there is no
visualiser and no IO."""
import numpy as np

import cupoch_b200 as cph
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth

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
    voxel_length = 2.0 / 256
    volume = cph.integration.ScalableTSDFVolume(voxel_length=voxel_length, sdf_trunc=0.04,
                                                color_type=cph.integration.TSDFVolumeColorType.RGB8)
    rng = np.random.default_rng(0)
    for _, E in cams:
        depth = cph.geometry.Image(np.round(depth_map(K, E) * 1000).astype(np.uint16))  # millimetres, as a sensor gives
        color = cph.geometry.Image(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        rgbd = cph.geometry.RGBDImage.create_from_color_and_depth(color, depth, depth_trunc=4.0, convert_rgb_to_intensity=False)
        volume.integrate(rgbd, intrinsic, E)
    units, capacity, nbytes = volume.info()
    print("units:", units, "of 16^3 voxels (pool capacity %d), %.1f MB on the device" % (capacity, nbytes / 1e6))
    print("a dense 256^3 RGB8 UniformTSDFVolume over the same 2 m box: %.1f MB" % (256 ** 3 * 20 / 1e6))
    print("extract_point_cloud:", len(volume.extract_point_cloud()), "points with normals")
    print("extract_voxel_point_cloud:", len(volume.extract_voxel_point_cloud()), "voxels in the band")


if __name__ == "__main__":
    main()
