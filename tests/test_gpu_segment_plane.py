"""GPU parity of PointCloud::SegmentPlane (csrc/segment.cu) through the Python mirror: bit-identical to the CPU
oracle (best iteration, inlier indices, plane, fitness, inlier_rmse) with the seeds the mirror draws from libc rand(),
plus the reference's known-answer test and the quirks of segmentation.cu:187-267."""
import ctypes as C
import json
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from conftest import ROOT
from cupoch_b200.testing import datagen

_libc = C.CDLL(None)
_libc.rand.restype = C.c_int


def seeds_after(seed, T):
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


def check_equal(seg, pc, pts, thr, ransac_n, T, seed):
    """srand(seed), run the product, and compare with the oracle given the same T rand() draws"""
    seeds = seeds_after(seed, T)
    _libc.srand(C.c_uint(seed))
    plane, idx = pc.segment_plane(thr, ransac_n, T)
    best, fit, rmse = pc.last_ransac_stats
    o_plane, o_idx, o_best, o_fit, o_rmse = seg.segment_plane(pts, thr, ransac_n, seeds)
    assert best == o_best
    np.testing.assert_array_equal(idx.cpu(), o_idx)
    np.testing.assert_array_equal(plane, o_plane)
    assert np.float32(fit) == o_fit and np.float32(rmse) == o_rmse
    return plane, idx


def test_golden_known_plane(seg, known_plane):
    g = known_plane
    pts = np.array(g["points"], np.float32)
    pc = cph.geometry.PointCloud(pts)
    for s in (1, 2, 77):
        plane, idx = check_equal(seg, pc, pts, g["distance_threshold"], g["ransac_n"], g["num_iterations"], s)
        assert idx.cpu().tolist() == g["inliers"]
        np.testing.assert_array_equal(pc.select_by_index(idx).points.cpu(), pts)


_SCENES = {}


def _scene(n):
    if n not in _SCENES:
        _SCENES[n] = datagen.plane_scene(n, 11)
    return _SCENES[n]


@pytest.mark.parametrize("n", [1000, 100_000, 1_000_000])
@pytest.mark.parametrize("T", [1, 10, 100, 1000])
def test_plane_scene_vs_oracle(seg, n, T):
    pts = _scene(n)
    plane, idx = check_equal(seg, cph.geometry.PointCloud(pts), pts, 0.01, 3, T, 1000 + T)
    if T >= 100:
        assert abs(abs(plane[2]) - 1) < 1e-3  # the ground


def test_20m_fitness_rounds(seg):
    """above 2^24 points (float)count / (float)n no longer separates neighbouring counts: ties go to the rmse rule"""
    n = 20_000_000
    pts = datagen.plane_scene(n, 12)
    check_equal(seg, cph.geometry.PointCloud(pts), pts, 0.01, 3, 10, 5)


def test_consecutive_calls_continue_the_libc_stream(seg):
    pts = _scene(100_000)
    pc = cph.geometry.PointCloud(pts)
    seeds = seeds_after(21, 40)
    _libc.srand(C.c_uint(21))
    a = pc.segment_plane(0.01, 3, 20)
    b = pc.segment_plane(0.01, 3, 20)
    for (plane, idx), sd in ((a, seeds[:20]), (b, seeds[20:])):
        o_plane, o_idx, _, _, _ = seg.segment_plane(pts, 0.01, 3, sd)
        np.testing.assert_array_equal(plane, o_plane)
        np.testing.assert_array_equal(idx.cpu(), o_idx)


def test_run_to_run_bit_reproducible():
    pc = cph.geometry.PointCloud(_scene(1_000_000))
    out = []
    for _ in range(2):
        _libc.srand(C.c_uint(9))
        plane, idx = pc.segment_plane(0.01, 3, 200)
        out.append((plane, idx.cpu(), pc.last_ransac_stats))
    np.testing.assert_array_equal(out[0][0], out[1][0])
    np.testing.assert_array_equal(out[0][1], out[1][1])
    assert out[0][2] == out[1][2]


def test_degenerate_cases_vs_oracle(seg):
    pts = datagen.plane_scene(5000, 3)
    pc = cph.geometry.PointCloud(pts)
    for ransac_n in (2, 5001):  # guards: zero plane, no inliers, no rand() drawn
        plane, idx = pc.segment_plane(0.01, ransac_n, 10)
        assert not plane.any() and len(idx) == 0
    check_equal(seg, cph.geometry.PointCloud(pts[:4]), pts[:4], 0.01, 4, 10, 2)  # n == ransac_n
    plane, idx = check_equal(seg, pc, pts, 0.01, 3, 0, 1)  # no iteration: the zero plane keeps every point
    assert len(idx) == 5000
    for thr in (0.0, -1.0):
        plane, idx = check_equal(seg, pc, pts, thr, 3, 10, 3)
        assert len(idx) == 0 and not plane.any()
    i = np.arange(300, dtype=np.float32)[:, None]
    line = (i * np.array([1, 2, 3], np.float32)).astype(np.float32)
    check_equal(seg, cph.geometry.PointCloud(line), line, 0.01, 3, 20, 4)
    assert cph.geometry.PointCloud(line).segment_plane(0.01, 3, 5)[1] is not None
    nanpts = pts.copy()
    nanpts[::7] = np.nan
    _, idx = check_equal(seg, cph.geometry.PointCloud(nanpts), nanpts, 0.01, 3, 50, 6)
    assert not np.isin(idx.cpu(), np.arange(0, 5000, 7)).any()


def test_select_complement_removes_the_plane(seg):
    pts = _scene(100_000)
    pc = cph.geometry.PointCloud(pts)
    _libc.srand(C.c_uint(31))
    plane, idx = pc.segment_plane(0.01, 3, 100)
    rest = pc.select_by_index(idx, invert=True)
    mask = np.ones(len(pts), bool)
    mask[idx.cpu()] = False
    np.testing.assert_array_equal(rest.points.cpu(), pts[mask])
    assert len(rest) + len(idx) == len(pts)
