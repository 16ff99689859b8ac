"""GPU: integration.ScalableTSDFVolume (csrc/stsdf.cu) against oracle/stsdf.c bit for bit -- the units' keys and slot
order, the tsdf / weight / colour blocks and both extractions.

- The reference's five real frames (tests/golden/tsdf_rgbd_known.npz) and synthetic sphere views for every colour type;
- a camera that sees only part of the allocated units;
- growth: map_size 1 and 100000 give the same bits, and repeats are bit-identical;
- reset, the argument rules, and a rejected frame (a unit key out of range) that leaves every bit unchanged;
- units only near the surface, and the device bytes against a UniformTSDFVolume over the same box."""
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import stsdf_py as S
from oracle import tsdf_py as T

G, CAM, I = cph.geometry, cph.camera, cph.integration
CT = I.TSDFVolumeColorType
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


def state(vol):
    keys, tw, col = vol.units()
    if len(keys) == 0:
        return np.zeros(0, np.uint64), np.zeros((0, 4096, 2), np.float32), None
    return keys.cpu(), tw.cpu(), (col.cpu() if col is not None else None)


def check_same(vol, ref):
    k, tw, col = state(vol)
    rk, rtw, rcol = ref.units()
    assert np.array_equal(k, rk)
    assert same(tw, rtw)
    if col is not None:
        assert same(col, rcol)
    p, n, c = ref.extract_point_cloud()
    pc = vol.extract_point_cloud()
    assert same(rows(pc, "points"), p) and same(rows(pc, "normals"), n)
    assert same(rows(pc, "colors"), c if c is not None else np.zeros((0, 3), np.float32))
    vp, vc = ref.extract_voxel_point_cloud()
    vpc = vol.extract_voxel_point_cloud()
    assert same(rows(vpc, "points"), vp) and same(rows(vpc, "colors"), vc)
    return len(k), len(p), len(vp)


def sphere_frames(n, w, h, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for K, E in ring_cameras(n, w, h):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        out.append((K, E, d16, rng.integers(0, 256, (h, w, 3), dtype=np.uint8)))
    return out


def integrate_both(vol, ref, frames, ct, w, h):
    for K, E, d16, rgb in frames:
        im = G.RGBDImage.create_from_color_and_depth(G.Image(rgb), G.Image(d16), 1000.0, 4.0, ct == CT.Gray32)
        depth = T.depth_to_float(d16, 1000.0, 4.0)
        col = T.intensity(rgb) if ct == CT.Gray32 else rgb
        vol.integrate(im, intrinsic(K, w, h), E)
        ref.integrate(depth, col, K, E)


def test_real_frames_match_oracle_and_stay_near_the_surface():
    z = np.load(GOLDEN)
    K = CAM.PinholeCameraIntrinsic(CAM.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    vol = I.ScalableTSDFVolume(4.0 / 512, 0.04, CT.RGB8)
    ref = S.Volume(4.0 / 512, 0.04, S.RGB8)
    rng = np.random.default_rng(5)
    for i in range(5):
        rgb = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(rgb), G.Image(z["depth"][i]), 1000.0, 4.0, False)
        vol.integrate(im, K, z["extrinsics"][i])
        ref.integrate(T.depth_to_float(z["depth"][i], 1000.0, 4.0), rgb, K.intrinsic_matrix, z["extrinsics"][i])
        units, npts, nvox = check_same(vol, ref)
    assert npts > 1000 and nvox > 1000
    units, cap, nbytes = vol.info()
    # every allocated unit holds a point of some frame within sdf_trunc; the whole box of units is much larger
    ku = S.unpack(ref.units()[0])
    box = np.prod(ku.max(0) - ku.min(0) + 1)
    assert units == len(ku) and units < 0.5 * box
    assert nbytes >= units * 4096 * 20


@pytest.mark.parametrize("ct", [CT.NoColor, CT.RGB8, CT.Gray32])
def test_sphere_views_every_colour_type(ct):
    w, h = 96, 72
    vol = I.ScalableTSDFVolume(1.0 / 64, 0.04, ct, 3)
    ref = S.Volume(1.0 / 64, 0.04, int(ct), 3)
    integrate_both(vol, ref, sphere_frames(6, w, h), ct, w, h)
    units, npts, nvox = check_same(vol, ref)
    assert units > 50 and npts > 1000
    # a camera that sees only part of the allocated units
    K, E = ring_cameras(6, w, h)[0]
    E2 = E.copy()
    E2[:3, 3] += np.float32([0.3, 0.0, -0.8])
    integrate_both(vol, ref, [(K, E2, np.round(sphere_depth(K, E2, w, h, 0.6) * 1000).astype(np.uint16),
                                np.full((h, w, 3), 7, np.uint8))], ct, w, h)
    check_same(vol, ref)


def test_map_size_and_repeats_change_no_bit():
    w, h = 80, 60
    frames = sphere_frames(4, w, h, 3)
    outs = []
    for map_size in (1, 100000, 1):
        vol = I.ScalableTSDFVolume(1.0 / 64, 0.05, CT.RGB8, 4, map_size)
        ref = S.Volume(1.0 / 64, 0.05, S.RGB8, 4)
        integrate_both(vol, ref, frames, CT.RGB8, w, h)
        check_same(vol, ref)
        k, tw, col = state(vol)
        outs.append((k, tw, col, rows(vol.extract_point_cloud(), "normals")))
        if map_size == 1:
            assert vol.info()[1] >= vol.info()[0] > 1  # grew from one slot
    for o in outs[1:]:
        assert np.array_equal(o[0], outs[0][0]) and same(o[1], outs[0][1]) and same(o[2], outs[0][2]) and same(o[3], outs[0][3])


def test_reset_errors_and_a_rejected_frame_leaves_the_volume_unchanged():
    w, h = 64, 48
    frames = sphere_frames(2, w, h, 4)
    vol = I.ScalableTSDFVolume(1.0 / 64, 0.04, CT.RGB8, 4, 1)
    ref = S.Volume(1.0 / 64, 0.04, S.RGB8, 4)
    integrate_both(vol, ref, frames[:1], CT.RGB8, w, h)
    before = state(vol)
    K, E, d16, rgb = frames[1]
    far = E.copy()
    far[:3, 3] += np.float32([0, 0, -1e6])  # the points land a million metres away: keys past 2^20 units of 0.25 m
    im = G.RGBDImage.create_from_color_and_depth(G.Image(rgb), G.Image(d16), 1000.0, 4.0, False)
    with pytest.raises(_lib.CphbError):
        vol.integrate(im, intrinsic(K, w, h), far)
    with pytest.raises(_lib.CphbError):
        vol.integrate(im, intrinsic(K, w, h), np.zeros((4, 4), np.float32))
    with pytest.raises(_lib.CphbError):  # the wrong colour format for RGB8
        vol.integrate(G.RGBDImage.create_from_color_and_depth(G.Image(rgb), G.Image(d16)), intrinsic(K, w, h), E)
    after = state(vol)
    assert np.array_equal(before[0], after[0]) and same(before[1], after[1]) and same(before[2], after[2])
    check_same(vol, ref)
    with pytest.raises(NotImplementedError):
        vol.extract_triangle_mesh()
    for bad in (dict(voxel_length=0.0), dict(sdf_trunc=-1.0), dict(depth_sampling_stride=0), dict(map_size=0)):
        args = dict(voxel_length=0.01, sdf_trunc=0.04, color_type=CT.NoColor)
        args.update(bad)
        with pytest.raises(_lib.CphbError):
            I.ScalableTSDFVolume(**args)
    vol.reset()
    assert vol.info()[0] == 0 and len(vol.extract_point_cloud()) == 0 and len(vol.extract_voxel_point_cloud()) == 0
    ref.reset()
    integrate_both(vol, ref, frames[1:], CT.RGB8, w, h)
    check_same(vol, ref)
    assert "ScalableTSDFVolume with color" in repr(vol)
