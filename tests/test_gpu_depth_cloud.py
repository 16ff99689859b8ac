"""GPU: geometry.PointCloud.create_from_depth_image / create_from_rgbd_image (csrc/depth_cloud.cu) against
oracle/depth_cloud.c bit for bit -- points, normals, colours and row order.

- uint16 and float32 depth at strides 1, 3 and 4 on odd image sizes, with a non-rigid extrinsic;
- RGB8 and Gray32 colour, depth_cutoff, compute_normals, both project_valid_depth_only settings;
- the reference's five real depth frames (tests/golden/tsdf_rgbd_known.npz);
- repeats, the argument rules, and two synthetic depth frames whose clouds feed estimate_normals and point-to-plane
  registration_icp, which recovers the relative camera pose."""
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing.datagen import gt_transform, ring_cameras, sphere_depth
from oracle import depth_cloud_py as D
from oracle import tsdf_py as T

G, CAM, R = cph.geometry, cph.camera, cph.registration
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsdf_rgbd_known.npz")


def bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def intrinsic(K, w, h):
    K = np.asarray(K, np.float32)
    return CAM.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])


def rows(pc, attr):
    a = getattr(pc, attr)
    return a.cpu() if len(pc) and a is not None else np.zeros((0, 3), np.float32)


def non_rigid(seed):
    rng = np.random.default_rng(seed)
    E = np.eye(4, dtype=np.float32)
    E[:3, :3] = np.eye(3) + rng.uniform(-0.3, 0.3, (3, 3))
    E[:3, 3] = rng.uniform(-1, 1, 3)
    return E


def scene(w, h, seed):
    """a sphere view with holes and noise: float32 metres and the matching uint16 millimetres"""
    K, E = ring_cameras(5, w, h)[seed % 5]
    d = sphere_depth(K, E, w, h, 0.8)
    rng = np.random.default_rng(seed)
    d = np.where(rng.random(d.shape) < 0.05, 0, d * rng.uniform(0.99, 1.01, d.shape)).astype(np.float32)
    return K, E, d, np.round(d * 1000).astype(np.uint16)


@pytest.mark.parametrize("stride", [1, 3, 4])
@pytest.mark.parametrize("dtype", ["uint16", "float32"])
def test_depth_image_matches_oracle(dtype, stride):
    w, h = 101, 77
    K, E, d, raw = scene(w, h, stride)
    img = raw if dtype == "uint16" else d
    for ext in (E, non_rigid(stride)):
        for scale, trunc in ((1000.0, 1000.0), (999.5, 2.5)):
            pc = G.PointCloud.create_from_depth_image(G.Image(img), intrinsic(K, w, h), ext, scale, trunc, stride)
            rp, _, _ = D.depth_to_points(img, K, ext, scale, trunc, stride)
            assert len(rp) > 50 and same(rows(pc, "points"), rp)
            assert pc.normals is None and pc.colors is None


@pytest.mark.parametrize("valid_only", [True, False])
@pytest.mark.parametrize("colour", ["rgb8", "gray32"])
def test_rgbd_image_matches_oracle(colour, valid_only):
    w, h = 97, 71
    K, E, d, raw = scene(w, h, 7)
    rng = np.random.default_rng(3)
    rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    im = G.RGBDImage.create_from_color_and_depth(G.Image(rgb), G.Image(raw), 1000.0, 4.0, colour == "gray32")
    depth = T.depth_to_float(raw, 1000.0, 4.0)
    col = T.intensity(rgb) if colour == "gray32" else rgb
    assert same(np.asarray(im.depth), depth)
    for ext in (E, non_rigid(11)):
        for cutoff in (-1.0, 2.0):
            for normals in (False, True):
                pc = G.PointCloud.create_from_rgbd_image(im, intrinsic(K, w, h), ext, valid_only, cutoff, normals)
                rp, rn, rc = D.depth_to_points(depth, K, ext, color=col, depth_cutoff=cutoff, compute_normals=normals,
                                               project_valid_depth_only=valid_only)
                assert len(rp) > 50
                assert same(rows(pc, "points"), rp) and same(rows(pc, "colors"), rc)
                if normals:
                    assert same(rows(pc, "normals"), rn)
                else:
                    assert pc.normals is None
                if not valid_only:
                    assert len(pc) == w * h and np.isnan(rp).any()


def test_host_rgbd_wrapper_and_real_frames():
    z = np.load(GOLDEN)
    K = CAM.PinholeCameraIntrinsic(CAM.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    rng = np.random.default_rng(5)
    for i in range(5):
        gray = rng.uniform(0, 1, (480, 640)).astype(np.float32)
        depth = T.depth_to_float(z["depth"][i], 1000.0, 4.0)
        im = G.RGBDImage(G.Image(gray), G.Image(depth))  # host images, uploaded as they are
        pc = G.PointCloud.create_from_rgbd_image(im, K, z["extrinsics"][i], compute_normals=True)
        rp, rn, rc = D.depth_to_points(depth, K.intrinsic_matrix, z["extrinsics"][i], color=gray, compute_normals=True)
        assert len(rp) > 100000
        assert same(rows(pc, "points"), rp) and same(rows(pc, "normals"), rn) and same(rows(pc, "colors"), rc)
        pd = G.PointCloud.create_from_depth_image(G.Image(z["depth"][i]), K, z["extrinsics"][i], 1000.0, 4.0, 4)
        assert same(rows(pd, "points"), D.depth_to_points(z["depth"][i], K.intrinsic_matrix, z["extrinsics"][i], 1000.0, 4.0, 4)[0])


def test_repeats_are_bit_identical_and_empty_frames_give_empty_clouds():
    w, h = 64, 48
    K, E, d, _ = scene(w, h, 2)
    im = G.RGBDImage(G.Image(d), G.Image(d))
    a = G.PointCloud.create_from_rgbd_image(im, intrinsic(K, w, h), E, True, -1.0, True)
    for _ in range(3):
        b = G.PointCloud.create_from_rgbd_image(im, intrinsic(K, w, h), E, True, -1.0, True)
        for attr in ("points", "normals", "colors"):
            assert same(rows(a, attr), rows(b, attr))
    zero = np.zeros((h, w), np.float32)
    assert len(G.PointCloud.create_from_depth_image(G.Image(zero), intrinsic(K, w, h))) == 0
    assert len(G.PointCloud.create_from_depth_image(G.Image(zero[:2, :2]), intrinsic(K, w, h), stride=3)) == 0


def test_argument_errors_raise():
    w, h = 8, 6
    K = intrinsic(np.eye(3) * 5, w, h)
    d = np.ones((h, w), np.float32)
    with pytest.raises(ValueError):
        G.PointCloud.create_from_depth_image(G.Image(np.ones((h, w), np.uint8)), K)
    with pytest.raises(ValueError):
        G.PointCloud.create_from_depth_image(G.Image(np.ones((h, w, 3), np.float32)), K)
    for bad in (dict(stride=0), dict(extrinsic=np.zeros((4, 4)))):
        with pytest.raises(_lib.CphbError):
            G.PointCloud.create_from_depth_image(G.Image(d), K, **bad)
    with pytest.raises(_lib.CphbError):
        G.PointCloud.create_from_depth_image(G.Image(d.astype(np.uint16)), K, depth_scale=0.5)
    with pytest.raises(_lib.CphbError):  # 3-channel float colour
        G.PointCloud.create_from_rgbd_image(G.RGBDImage(G.Image(np.ones((h, w, 3), np.float32)), G.Image(d)), K)
    with pytest.raises(_lib.CphbError):  # sizes differ
        G.PointCloud.create_from_rgbd_image(G.RGBDImage(G.Image(np.ones((h, w - 1), np.float32)), G.Image(d)), K)
    with pytest.raises(_lib.CphbError):
        G.PointCloud.create_from_rgbd_image(G.RGBDImage(G.Image(d), G.Image(d)), K, depth_cutoff=float("nan"))
    with pytest.raises(ValueError):  # the depth of an RGBDImage is float32
        G.PointCloud.create_from_rgbd_image(G.RGBDImage(G.Image(d), G.Image(d.astype(np.uint16))), K)


def scene_depth(K, E, w, h):
    """camera depth of a few spheres in front of a tilted wall (no continuous symmetry), world-to-camera E"""
    best = np.full((h, w), np.inf, np.float32)
    for c, r in (((0.0, 0.0, 0.0), 0.45), ((0.55, 0.35, 0.2), 0.25), ((-0.4, 0.45, -0.3), 0.3), ((0.1, -0.5, 0.35), 0.2)):
        T_c = np.eye(4, dtype=np.float32)
        T_c[:3, 3] = c
        d = sphere_depth(K, E @ T_c, w, h, r)
        best = np.where((d > 0) & (d < best), d, best)
    Ki = np.linalg.inv(np.asarray(K, np.float64))
    uu, vv = np.meshgrid(np.arange(w), np.arange(h))
    rays = np.stack([uu, vv, np.ones_like(uu)], -1) @ Ki.T
    Rm, t = np.asarray(E, np.float64)[:3, :3], np.asarray(E, np.float64)[:3, 3]
    nw, off = np.array([1.0, 0.3, 0.2]) / np.linalg.norm([1.0, 0.3, 0.2]), -0.9  # world plane nw . X = off
    nc = Rm @ nw  # in the camera: nc . x = off + nc . t
    wall = (off + nc @ t) / (rays @ nc)
    best = np.where((wall > 0) & (wall < best), wall, best)
    return np.where(np.isfinite(best), best, 0).astype(np.float32)


def test_depth_frames_feed_point_to_plane_icp():
    w, h = 320, 240
    K, E1 = ring_cameras(8, w, h)[0]
    dT = gt_transform((1.0, -1.5, 2.0), (0.02, -0.01, 0.015)).astype(np.float32)
    E2 = dT @ E1  # the second camera moved by dT in the first camera's frame
    cams = []
    for E in (E1, E2):
        d = scene_depth(K, E, w, h)
        im = G.RGBDImage(G.Image(d), G.Image(d))
        cams.append(G.PointCloud.create_from_rgbd_image(im, intrinsic(K, w, h)))  # camera-frame clouds
    tgt, src = cams
    assert len(src) > 20000 and len(tgt) > 20000
    tgt.estimate_normals(G.KDTreeSearchParamKNN(20))
    want = E1.astype(np.float64) @ np.linalg.inv(E2.astype(np.float64))  # camera 2 -> camera 1
    res = R.registration_icp(src, tgt, 0.1, np.eye(4), R.TransformationEstimationPointToPlane(), R.ICPConvergenceCriteria(1e-9, 1e-9, 60))
    err = np.asarray(res.transformation, np.float64) - want
    assert np.abs(err[:3, :3]).max() < 2e-3 and np.abs(err[:3, 3]).max() < 2e-3, (res.transformation, want)
    assert res.fitness > 0.8
