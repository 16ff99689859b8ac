"""CPU: the SegmentPlane restatement (oracle/segment_plane.c) -- pinned to the reference's known-answer test, its
sampler pinned to thrust itself (the toolkit's headers, CPP backend), its scoring / selection / refit checked against
an independent float64 numpy restatement, and every quirk of segmentation.cu:187-267 it mirrors."""
import ctypes as C
import json
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from cupoch_b200.testing import datagen

_libc = C.CDLL(None)
_libc.rand.restype = C.c_int


def libc_seeds(seed, T):
    """the seeds the reference draws: rand() once per iteration after srand(seed)"""
    _libc.srand(C.c_uint(seed))
    return np.array([_libc.rand() for _ in range(T)], np.int32)


@pytest.fixture(scope="module")
def seg():
    """the SegmentPlane restatement (oracle/segment_plane.c)"""
    from oracle import segment_plane_py
    segment_plane_py.build()
    return segment_plane_py


@pytest.fixture(scope="module")
def known_plane():
    """the reference's SegmentPlaneKnownPlane test (tests/golden/segment_plane_known.json, from tools/make_golden.py)"""
    with open(os.path.join(ROOT, "tests", "golden", "segment_plane_known.json")) as f:
        return json.load(f)["segment_plane_known"]


def test_golden_known_plane(seg, known_plane):
    g = known_plane
    pts = np.array(g["points"], np.float32)
    for s in (1, 2, 77):  # 1 = the default srand state of a fresh process
        seeds = libc_seeds(s, g["num_iterations"])
        plane, idx, best, fit, rmse = seg.segment_plane(pts, g["distance_threshold"], g["ransac_n"], seeds)
        assert idx.tolist() == g["inliers"]
        assert best >= 0 and fit == np.float32(1.0)
        # the five points satisfy x = y: plane ~ +-(1, -1, 0, 0) / sqrt(2)
        np.testing.assert_allclose(np.abs(plane), [0.5 ** 0.5, 0.5 ** 0.5, 0, 0], atol=1e-5)
        assert plane[0] * plane[1] < 0


def _thrust_include():
    for d in (os.environ.get("CUDA_HOME", ""), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "include", "thrust", "random.h")):
            return os.path.join(d, "include")
    return None


def test_sampler_matches_thrust(seg):
    inc = _thrust_include()
    if inc is None or shutil.which("g++") is None:
        pytest.skip("needs g++ and the CUDA toolkit's thrust headers")
    seeds = [0, 2147483647, 1, 2, 48271, 12345, 2147483646, 1 << 30] + libc_seeds(5, 12).tolist()
    assert len(seeds) == 20
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "pin")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + inc, "-DTHRUST_DEVICE_SYSTEM=THRUST_DEVICE_SYSTEM_CPP",
                               os.path.join(ROOT, "tests", "cpp", "thrust_ransac_pin.cpp"), "-o", exe])
        for n in (5, 1000, 65537):
            out = os.path.join(d, "out.i32")
            subprocess.check_call([exe, out, str(n)] + [str(s) for s in seeds])
            rec = np.fromfile(out, np.int32).reshape(len(seeds), n + 3)
            for t, s in enumerate(seeds):
                np.testing.assert_array_equal(seg.ransac_keys(s, n), rec[t, :n], err_msg="keys n=%d seed=%d" % (n, s))
            np.testing.assert_array_equal(seg.ransac_samples(n, seeds), rec[:, n:], err_msg="samples n=%d" % n)


def _np_hypotheses(P, thr, samples):
    """float64 restatement of every hypothesis: (plane or None, count, error sum / sqrt(count), band count)"""
    out = []
    for s in samples:
        p0, p1, p2 = P[s]
        nrm = np.cross(p1 - p0, p2 - p0)
        nn = np.linalg.norm(nrm)
        if nn == 0:
            out.append((None, 0, 0.0, 0))
            continue
        nrm = nrm / nn
        pl = np.append(nrm, -nrm @ p0)
        dist = np.abs(P @ pl[:3] + pl[3])
        inl = dist < thr
        c = int(inl.sum())
        band = int((np.abs(dist - thr) <= 1e-6 * thr).sum())
        out.append((pl, c, dist[inl].sum() / np.sqrt(c) if c else 0.0, band))
    return out


def _np_select(hyp):
    best, bc, br = -1, 0, 0.0
    for t, (pl, c, r, _) in enumerate(hyp):
        if pl is None or c == 0:
            continue
        if c > bc or (c == bc and r < br):
            best, bc, br = t, c, r
    return best


def _guard(hyp, best):
    """the winner must not be within reach of a competitor: no other count within the threshold-ambiguity bands, and
    on an equal count the error sums more than 1 float32 ulp apart"""
    _, cb, rb, bb = hyp[best]
    for t, (pl, c, r, band) in enumerate(hyp):
        if t == best or pl is None:
            continue
        if c + band >= cb - bb:
            assert c == cb and band == 0 and bb == 0, (t, c, cb)
            assert abs(r - rb) > np.spacing(np.float32(rb)), (t, r, rb)


@pytest.mark.parametrize("n,T,seed", [(3000, 50, 3), (20000, 200, 8)])
def test_vs_numpy_float64(seg, n, T, seed):
    pts = datagen.plane_scene(n, seed)
    thr = 0.01
    seeds = libc_seeds(seed, T)
    plane, idx, best, fit, rmse = seg.segment_plane(pts, thr, 3, seeds)
    samples = seg.ransac_samples(n, seeds)
    P = pts.astype(np.float64)
    hyp = _np_hypotheses(P, thr, samples)
    nb = _np_select(hyp)
    _guard(hyp, nb)
    assert best == nb
    pl, c, r, _ = hyp[nb]
    assert fit == np.float32(c) / np.float32(n)
    np.testing.assert_allclose(rmse, r, rtol=1e-5)
    dist = np.abs(P @ pl[:3] + pl[3])
    clear = np.abs(dist - thr) > 1e-6 * thr
    mine = np.zeros(n, bool)
    mine[idx] = True
    np.testing.assert_array_equal(mine[clear], (dist < thr)[clear])
    assert (np.diff(idx) > 0).all()
    # refit: least-squares plane of the final inliers (float64 eigen-decomposition)
    Q = P[idx]
    cen = Q.mean(0)
    w, V = np.linalg.eigh((Q - cen).T @ (Q - cen))
    nrm = V[:, 0] * np.sign(V[:, 0] @ plane[:3])
    np.testing.assert_allclose(plane[:3], nrm, atol=1e-5)
    np.testing.assert_allclose(plane[3], -nrm @ cen, atol=1e-5)
    assert abs(abs(plane[2]) - 1) < 1e-3  # the ground wins this scene


def _run(seg, pts, thr=0.01, ransac_n=3, T=20, seed=4):
    return seg.segment_plane(pts, thr, ransac_n, libc_seeds(seed, T))


def test_guards_zero_plane_no_inliers(seg):
    pts = datagen.plane_scene(500, 1)
    for args in ({"ransac_n": 2}, {"ransac_n": 0}, {"ransac_n": 501}):
        plane, idx, best, fit, rmse = _run(seg, pts, **args)
        assert not plane.any() and len(idx) == 0 and best == -1 and fit == 0 and rmse == 0
    plane, idx, best, _, _ = _run(seg, pts[:2])  # n < ransac_n
    assert not plane.any() and len(idx) == 0 and best == -1
    plane, idx, best, _, _ = _run(seg, pts[:5], ransac_n=5)  # n == ransac_n is enough
    assert best >= 0 and len(idx) >= 3


def test_no_iterations_every_point_is_an_inlier(seg):
    pts = datagen.plane_scene(500, 2)
    plane, idx, best, fit, rmse = _run(seg, pts, T=0)
    assert best == -1 and fit == 0 and rmse == 0
    np.testing.assert_array_equal(idx, np.arange(500))  # the zero plane: dist 0 < threshold
    assert np.linalg.norm(plane[:3]) == pytest.approx(1, abs=1e-6)


def test_non_positive_threshold_keeps_nothing(seg):
    pts = datagen.plane_scene(500, 3)
    for thr in (0.0, -0.5):
        plane, idx, best, fit, rmse = _run(seg, pts, thr=thr)
        assert best == -1 and len(idx) == 0 and not plane.any()


def test_collinear_points_every_hypothesis_skipped(seg):
    i = np.arange(200, dtype=np.float32)[:, None]
    pts = (i * np.array([1, 2, 3], np.float32)).astype(np.float32)  # exact integer multiples: every cross product is 0
    plane, idx, best, fit, rmse = _run(seg, pts, T=30)
    assert best == -1 and fit == 0
    np.testing.assert_array_equal(idx, np.arange(200))


def test_nan_points_are_never_inliers(seg):
    pts = datagen.plane_scene(2000, 5)
    pts[::7] = np.nan
    plane, idx, best, fit, rmse = _run(seg, pts, T=60)
    assert best >= 0 and np.isfinite(plane).all()
    assert not np.isin(idx, np.arange(0, 2000, 7)).any()
    _, idx0, _, _, _ = _run(seg, pts, T=0)
    np.testing.assert_array_equal(idx0, np.setdiff1d(np.arange(2000), np.arange(0, 2000, 7)))
