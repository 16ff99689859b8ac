"""GPU: integration.UniformTSDFVolume and geometry.RGBDImage (csrc/tsdf.cu) against oracle/tsdf.c bit for bit.

- The reference's five real RGB-D frames (tests/golden/tsdf_rgbd_known.npz): the tsdf / weight / colour planes after every
  frame, both extractions, the voxel grid and raycasts, and the reference test's counts and sums.
- Synthetic sphere views (16 per volume) at resolution 128 and 256 with all three colour types, one 512^3 volume with
  640 x 480 frames, cameras outside and inside the grid, an axis-aligned ray and project_valid_depth_only both ways.
- Reset, bit-identical repeats, a fixed launch count per call, the argument rules, the voxel grid's keys and one
  point-to-plane ICP against a raycast."""
import ctypes
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import tsdf_py as T

G, CAM, I = cph.geometry, cph.camera, cph.integration
CT = I.TSDFVolumeColorType
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsdf_rgbd_known.npz")


def bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def same_planes(vol, ref):
    tw, col = vol.planes()
    assert same(tw.cpu(), ref.tw)
    if col is not None:
        assert same(col.cpu(), ref.col)


def intrinsic(K, w, h):
    K = np.asarray(K, np.float32)
    return CAM.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])


def cloud(pc, with_colors=True):
    n = len(pc)
    z = np.zeros((0, 3), np.float32)
    return (pc.points.cpu() if n else z, pc.normals.cpu() if n and pc.has_normals() else z,
            pc.colors.cpu() if n and with_colors and pc.has_colors() else z)


def check_extractions(vol, ref):
    p, n, c = cloud(vol.extract_point_cloud())
    rp, rn, rc = ref.extract_point_cloud()
    assert same(p, rp) and same(n, rn)
    assert same(c, rc if rc is not None else np.zeros((0, 3), np.float32))
    vp = vol.extract_voxel_point_cloud()
    rvp, rvc = ref.extract_voxel_point_cloud()
    got = cloud(vp)
    assert same(got[0], rvp) and same(got[2], rvc)
    vg = vol.extract_voxel_grid()
    keys, cols = vg.get_voxels()
    rk, rcol, vs, org = ref.extract_voxel_grid()
    assert np.array_equal(keys, rk) and same(cols, rcol)
    assert vg.voxel_size == float(vs) and same(vg.origin, org)
    return len(rp), len(rvp)


def check_raycast(vol, ref, K, E, w, h, trunc):
    for valid in (True, False):
        p, n, c = cloud(vol.raycast(intrinsic(K, w, h), E, trunc, valid))
        rp, rn, rc = ref.raycast(K, E, w, h, trunc, valid)
        assert same(p, rp) and same(n, rn) and same(c, rc), valid
        if not valid:
            assert len(p) == w * h
    return len(rp)


def rgbd(depth_m, color, ct):
    """an RGBDImage of a metric float32 depth map: depth in millimetres as uint16 through CreateFromColorAndDepth"""
    d16 = np.round(np.asarray(depth_m) * 1000).astype(np.uint16)
    return G.RGBDImage.create_from_color_and_depth(G.Image(color), G.Image(d16), 1000.0, 100.0, ct == CT.Gray32), d16


def oracle_frame(d16, color, ct):
    d = T.depth_to_float(d16, 1000.0, 100.0)
    c = None if ct == CT.NoColor else (T.intensity(color) if ct == CT.Gray32 else color)
    return d, c


# ------------------------------------------------------------------------------------------------ real data
@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_real_data_matches_oracle_and_reference_values(golden):
    K = CAM.PinholeCameraIntrinsic(CAM.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    vol = I.UniformTSDFVolume(8.0, 200, 0.04, CT.RGB8)
    ref = T.Volume(8.0, 200, 0.04, T.RGB8)
    rng = np.random.default_rng(5)
    for i in range(5):
        color = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)  # the JPEG colours are not part of the fixture
        im = G.RGBDImage.create_from_color_and_depth(G.Image(color), G.Image(golden["depth"][i]), 1000.0, 4.0, False)
        d = T.depth_to_float(golden["depth"][i], 1000.0, 4.0)
        assert same(np.asarray(im.depth), d)
        vol.integrate(im, K, golden["extrinsics"][i])
        ref.integrate(d, color, K.intrinsic_matrix, golden["extrinsics"][i])
        same_planes(vol, ref)
    npts, nvox = check_extractions(vol, ref)
    assert npts == int(golden["points_count"]) and nvox == int(golden["voxel_count"])
    p, n, _ = cloud(vol.extract_point_cloud())
    assert np.all(np.abs(n.astype(np.float64).sum(0) - golden["normal_sum"]) <= golden["tolerance"])
    _, _, vc = cloud(vol.extract_voxel_point_cloud())
    assert np.all(np.abs(vc.astype(np.float64).sum(0) - golden["voxel_color_sum"]) <= golden["tolerance"])
    for i in (0, 4):
        assert check_raycast(vol, ref, K.intrinsic_matrix, golden["extrinsics"][i], 640, 480, 0.04) > 1000


# ------------------------------------------------------------------------------------------------ synthetic views
def views(n, w, h, radius=2.5):
    return ring_cameras(n, w, h, radius)


@pytest.mark.parametrize("res", [128, 256])
@pytest.mark.parametrize("ct", [CT.NoColor, CT.RGB8, CT.Gray32])
def test_sphere_views_match_oracle(res, ct):
    w, h = 160, 120
    length, trunc = 2.0, 0.06
    vol = I.UniformTSDFVolume(length, res, trunc, ct, origin=(0.01, -0.02, 0.03))
    ref = T.Volume(length, res, trunc, int(ct), origin=(0.01, -0.02, 0.03))
    rng = np.random.default_rng(res + int(ct))
    cams = views(16, w, h)
    for K, E in cams:
        color = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        im, d16 = rgbd(sphere_depth(K, E, w, h, 0.6), color, ct)
        vol.integrate(im, intrinsic(K, w, h), E)
        d, c = oracle_frame(d16, color, ct)
        ref.integrate(d, c, K, E)
        same_planes(vol, ref)
    npts, _ = check_extractions(vol, ref)
    assert npts > 1000
    for K, E in cams[:3]:  # cameras outside the grid
        assert check_raycast(vol, ref, K, E, w, h, trunc) > 0.2 * w * h
    Ki, Ei = ring_cameras(1, w, h, 0.9)[0]  # inside the grid ([-1, 1]^3), outside the sphere
    assert check_raycast(vol, ref, Ki, Ei, w, h, trunc) > 0.2 * w * h


def test_axis_aligned_rays_and_a_camera_far_outside():
    w, h, res, length, trunc = 161, 121, 128, 2.0, 0.06
    vol = I.UniformTSDFVolume(length, res, trunc, CT.NoColor)
    ref = T.Volume(length, res, trunc)
    for K, E in views(8, w, h):
        im, d16 = rgbd(sphere_depth(K, E, w, h, 0.6), np.zeros((h, w, 3), np.uint8), CT.NoColor)
        vol.integrate(im, intrinsic(K, w, h), E)
        ref.integrate(*oracle_frame(d16, None, CT.NoColor), K, E)
    K = np.float32([[100, 0, 80], [0, 100, 60], [0, 0, 1]])  # pixel (80, 60) looks exactly along +x
    for dist in (2.5, 30.0):
        E = np.zeros((4, 4), np.float32)
        E[0, 1] = E[1, 2] = E[2, 0] = E[3, 3] = 1  # camera x, y, z = world y, z, x
        E[2, 3] = dist
        check_raycast(vol, ref, K, E, w, h, trunc)
        p, _, _ = cloud(vol.raycast(intrinsic(K, w, h), E, trunc, False))
        # the central ray hits the sphere's front at x = -0.6 (the reference's [0, length] box would start it past it)
        assert abs(p[60 * w + 80, 0] + 0.6) < 0.02 and p[60 * w + 80, 1] == 0 and p[60 * w + 80, 2] == 0


def test_res512_with_640x480_frames():
    w, h = 640, 480
    vol = I.UniformTSDFVolume(2.0, 512, 0.03, CT.RGB8)
    ref = T.Volume(2.0, 512, 0.03, T.RGB8)
    rng = np.random.default_rng(9)
    for K, E in views(2, w, h):
        color = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        im, d16 = rgbd(sphere_depth(K, E, w, h, 0.6), color, CT.RGB8)
        vol.integrate(im, intrinsic(K, w, h), E)
        ref.integrate(*oracle_frame(d16, color, CT.RGB8), K, E)
    same_planes(vol, ref)
    check_extractions(vol, ref)
    K, E = views(2, w, h)[0]
    check_raycast(vol, ref, K, E, w, h, 0.03)


# ------------------------------------------------------------------------------------------------ properties
@pytest.fixture(scope="module")
def sphere_volume():
    w, h = 160, 120
    vol = I.UniformTSDFVolume(2.0, 128, 0.06, CT.RGB8)
    rng = np.random.default_rng(1)
    for K, E in views(8, w, h):
        im, _ = rgbd(sphere_depth(K, E, w, h, 0.6), rng.integers(0, 256, (h, w, 3), dtype=np.uint8), CT.RGB8)
        vol.integrate(im, intrinsic(K, w, h), E)
    return vol


def test_repeats_are_bit_identical_and_launch_counts_fixed(sphere_volume):
    L = _lib.lib()
    K, E = views(8, 160, 120)[0]
    calls = [lambda v: v.extract_point_cloud(), lambda v: v.extract_voxel_point_cloud(), lambda v: v.extract_voxel_grid(),
             lambda v: v.raycast(intrinsic(K, 160, 120), E, 0.06, True), lambda v: v.raycast(intrinsic(K, 160, 120), E, 0.06, False)]

    def rows(x):
        return x.get_voxels() if isinstance(x, G.VoxelGrid) else cloud(x)

    for f in calls:
        a, b = rows(f(sphere_volume)), rows(f(sphere_volume))
        assert all(np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)) for x, y in zip(a, b))
        assert len(a[0]) > 0
    # every C-ABI call launches the same kernels whatever the data: a full volume and an empty one, sizing and writing
    empty = I.UniformTSDFVolume(2.0, 128, 0.06, CT.RGB8)
    from cupoch_b200.utility import DeviceArray
    out = [DeviceArray((200000, 3), np.float32) for _ in range(3)]
    keys = DeviceArray((200000, 3), np.int32)
    n = ctypes.c_size_t(0)
    for fn, args in ((L.cphb_tsdf_extract_points, (None, None, None, 0)),
                     (L.cphb_tsdf_extract_points, (out[0].ptr, out[1].ptr, out[2].ptr, 200000)),
                     (L.cphb_tsdf_extract_voxels, (None, None, None, 0)),
                     (L.cphb_tsdf_extract_voxels, (keys.ptr, out[0].ptr, out[1].ptr, 200000))):
        counts = []
        for vol in (sphere_volume, empty):
            n0 = L.cphb_launch_count()
            _lib.check(fn(vol._h, *args, ctypes.byref(n), None))
            counts.append(L.cphb_launch_count() - n0)
        assert counts[0] == counts[1] and counts[0] > 0, counts


def test_reset_then_extract_is_empty():
    vol = I.UniformTSDFVolume(2.0, 64, 0.06, CT.Gray32)
    K, E = views(1, 160, 120)[0]
    im, _ = rgbd(sphere_depth(K, E, 160, 120, 0.6), np.zeros((120, 160, 3), np.uint8), CT.Gray32)
    vol.integrate(im, intrinsic(K, 160, 120), E)
    assert len(vol.extract_voxel_grid()) > 0
    vol.reset()
    assert len(vol.extract_point_cloud()) == 0 and len(vol.extract_voxel_point_cloud()) == 0 and len(vol.extract_voxel_grid()) == 0
    assert len(vol.raycast(intrinsic(K, 160, 120), E, 0.06)) == 0
    tw, col = vol.planes()
    assert not tw.cpu().any() and np.all(col.cpu() == 1.0)


def test_voxel_grid_keys_sorted_unique_and_hold_the_points(sphere_volume):
    vg = sphere_volume.extract_voxel_grid()
    k, _ = vg.get_voxels()
    packed = (k[:, 0].astype(np.int64) << 40) | (k[:, 1].astype(np.int64) << 20) | k[:, 2]
    assert len(k) > 1000 and np.all(np.diff(packed) > 0)
    p, _, _ = cloud(sphere_volume.extract_point_cloud())
    assert vg.check_if_included(p).all()


def test_argument_rules_raise():
    for args in [(2.0, 1, 0.1), (2.0, 1291, 0.1), (0.0, 64, 0.1), (np.inf, 64, 0.1), (2.0, 64, 0.0), (2.0, 64, np.nan), (-1.0, 64, 0.1)]:
        with pytest.raises(_lib.CphbError):
            I.UniformTSDFVolume(*args, CT.NoColor)
    vol = I.UniformTSDFVolume(2.0, 64, 0.06, CT.RGB8)
    K, E = views(1, 160, 120)[0]
    d = np.ones((120, 160), np.uint16)
    ok = G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((120, 160, 3), np.uint8)), G.Image(d), convert_rgb_to_intensity=False)
    with pytest.raises(_lib.CphbError):  # the image does not match the intrinsic
        vol.integrate(ok, intrinsic(K, 161, 120), E)
    gray = G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((120, 160, 3), np.uint8)), G.Image(d))
    with pytest.raises(_lib.CphbError):  # RGB8 needs uint8 RGB colour
        vol.integrate(gray, intrinsic(K, 160, 120), E)
    with pytest.raises(_lib.CphbError):
        vol.raycast(intrinsic(K, 160, 120), E, 0.0)
    with pytest.raises(ValueError):
        G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((10, 10, 3), np.uint8)), G.Image(d))
    with pytest.raises(_lib.CphbError):
        G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((120, 160, 3), np.uint8)), G.Image(d), depth_scale=0.5)


def test_depth_trunc_is_truncated_to_int():
    d = np.array([[1999, 2000, 2499, 2500, 0]], np.uint16)
    im = G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((1, 5), np.uint8)), G.Image(d), 1000.0, 2.5)
    assert same(np.asarray(im.depth), T.depth_to_float(d, 1000.0, 2.5))
    assert np.asarray(im.depth).tolist() == [[np.float32(1.999), 0.0, 0.0, 0.0, 0.0]]


# ------------------------------------------------------------------------------------------------ ICP against a raycast
def test_point_to_plane_icp_against_raycast_recovers_the_pose():
    w, h, res = 320, 240, 256
    centres = np.float32([[0, 0, 0], [0.45, 0.1, -0.2], [-0.2, 0.5, 0.25]])
    radii = (0.35, 0.2, 0.15)

    def depth(K, E):
        out = np.zeros((h, w), np.float32)
        for c, r in zip(centres, radii):
            Ec = E.copy()
            Ec[:3, 3] = E[:3, :3] @ c + E[:3, 3]
            d = sphere_depth(K, Ec, w, h, r)
            out = np.where((d > 0) & ((out == 0) | (d < out)), d, out)
        return out

    vol = I.UniformTSDFVolume(2.0, res, 0.04, CT.NoColor)
    cams = views(12, w, h)
    for K, E in cams:
        im, _ = rgbd(depth(K, E), np.zeros((h, w, 3), np.uint8), CT.NoColor)
        vol.integrate(im, intrinsic(K, w, h), E)
    K, E = cams[0]
    tgt = vol.raycast(intrinsic(K, w, h), E, 0.04)
    # the source: the analytic surface seen from the same view, back-projected, every 4th pixel, then moved by T^-1
    d = depth(K, E)
    v, u = np.nonzero(d[::2, ::2] > 0)
    v, u = v * 2, u * 2
    z = d[v, u].astype(np.float64)
    Ki = np.linalg.inv(K.astype(np.float64))
    cam_pts = (np.stack([u, v, np.ones_like(u)], 1) @ Ki.T) * z[:, None]
    Ed = E.astype(np.float64)
    world = (cam_pts - Ed[:3, 3]) @ Ed[:3, :3]
    from cupoch_b200.testing import datagen
    Tgt = datagen.gt_transform((1.0, -1.5, 2.0), (0.02, -0.01, 0.015)).astype(np.float64)  # degrees, metres
    src = ((world - Tgt[:3, 3]) @ Tgt[:3, :3]).astype(np.float32)  # T^-1 world
    R = cph.registration
    res_ = R.registration_icp(G.PointCloud(src), tgt, 0.05, np.eye(4), R.TransformationEstimationPointToPlane(),
                              R.ICPConvergenceCriteria(1e-9, 1e-9, 60))
    Tr = res_.transformation.astype(np.float64)
    dt = np.linalg.norm(Tr[:3, 3] - Tgt[:3, 3])
    ang = np.degrees(np.arccos(np.clip((np.trace(Tr[:3, :3] @ Tgt[:3, :3].T) - 1) / 2, -1, 1)))
    assert dt < 2e-3 and ang < 0.2, (dt, ang, res_.fitness)
