"""CPU: the ScalableTSDFVolume restatement (oracle/stsdf.c) against analytic scenes and the uniform volume's oracle.

- Units: every allocated unit lies within sdf_trunc of some strided depth point, and slots are ordered by the frame
  that first touched them, then by ascending key.
- Where a scalable and a uniform grid coincide (power-of-two voxel length, origin on the unit lattice) both give the
  same voxels: equal weights and tsdf within float32 rounding, and both extractions put a sphere on its surface.
"""
import numpy as np

from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import depth_cloud_py as D
from oracle import stsdf_py as S
from oracle import tsdf_py as T

W, H, R = 80, 60, 0.6


def frames(n):
    return [(K, E, sphere_depth(K, E, W, H, R)) for K, E in ring_cameras(n, W, H)]


def test_units_are_near_the_points_and_ordered_by_frame_then_key():
    vl, trunc, stride = 1.0 / 64, 0.04, 4
    U = vl * 16
    vol = S.Volume(vl, trunc, S.NO_COLOR, stride)
    seen = 0
    allowed = set()
    for K, E, d in frames(3):
        vol.integrate(d, None, K, E)
        keys = vol.units()[0]
        new = keys[seen:]
        assert np.all(np.diff(new.astype(np.uint64)) > 0)  # ascending within the frame
        p, _, _ = D.depth_to_points(d, K, E, stride=stride)
        lo, hi = np.floor((p - trunc) / U).astype(int), np.floor((p + trunc) / U).astype(int)
        for a, b in zip(lo, hi):
            for x in range(a[0], b[0] + 1):
                for y in range(a[1], b[1] + 1):
                    for z in range(a[2], b[2] + 1):
                        allowed.add((x, y, z))
        assert {tuple(k) for k in S.unpack(keys)} == allowed
        seen = len(keys)
    assert len(np.unique(keys)) == len(keys)


def test_scalable_and_uniform_grids_coincide():
    vl, trunc, res = 1.0 / 64, 0.05, 128  # length 2: uniform voxel k has centre vl (k - 64) + vl / 2, unit key (k - 64) // 16
    uni = T.Volume(2.0, res, trunc, T.NO_COLOR)
    sc = S.Volume(vl, trunc, S.NO_COLOR, 1)
    for K, E, d in frames(4):
        uni.integrate(d, None, K, E)
        sc.integrate(d, None, K, E)
    keys, tw, _ = sc.units()
    ku = S.unpack(keys)
    t = np.arange(4096)
    local = np.stack([t >> 8, (t >> 4) & 15, t & 15], 1)
    g = ku[:, None, :] * 16 + local[None] + res // 2  # the uniform index of every scalable voxel
    inside = np.all((g >= 0) & (g < res), 2)
    gi = g[inside]
    utw = uni.tw.reshape(res, res, res, 2)[gi[:, 0], gi[:, 1], gi[:, 2]]
    stw = tw[inside]
    same_w = utw[:, 1] == stw[:, 1]
    assert same_w.mean() > 0.999
    both = same_w & (stw[:, 1] > 0)
    assert both.sum() > 10000
    assert np.abs(utw[both, 0] - stw[both, 0]).max() < 1e-4
    # every band voxel of the uniform volume (near the surface) lies in an allocated unit
    utw_all = uni.tw.reshape(res, res, res, 2)
    bi = np.argwhere((utw_all[..., 1] > 0) & (np.abs(utw_all[..., 0]) < 0.98))
    assert len(bi) > 1000
    assert {tuple(k) for k in np.floor_divide(bi - res // 2, 16)} <= {tuple(k) for k in ku}
    p, n, _ = sc.extract_point_cloud()
    up, _, _ = uni.extract_point_cloud()
    assert abs(len(p) - len(up)) < 0.02 * len(up)
    assert np.abs(np.linalg.norm(p.astype(np.float64), axis=1) - R).max() < 1.5 * vl
    assert np.abs(np.linalg.norm(n, axis=1) - 1).max() < 1e-5
    vp, vc = sc.extract_voxel_point_cloud()
    assert np.abs(np.linalg.norm(vp.astype(np.float64), axis=1) - R).max() < trunc + vl
    assert np.all((vc >= 0) & (vc <= 1))


def test_rejected_frame_and_reset():
    vol = S.Volume(1.0 / 64, 0.04, S.RGB8, 4)
    K, E, d = frames(1)[0]
    rgb = np.zeros((H, W, 3), np.uint8)
    vol.integrate(d, rgb, K, E)
    before = vol.units()
    far = E.copy()
    far[:3, 3] += np.float32([0, 0, -1e6])
    try:
        vol.integrate(d, rgb, K, far)
        raised = False
    except ValueError:
        raised = True
    assert raised
    after = vol.units()
    for a, b in zip(before, after):
        assert np.array_equal(a, b)
    vol.reset()
    assert len(vol.units()[0]) == 0 and len(vol.extract_point_cloud()[0]) == 0
