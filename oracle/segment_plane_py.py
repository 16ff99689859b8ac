"""ctypes loader for the SegmentPlane restatement (oracle/segment_plane.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --segment-plane, never by the
product package cupoch_b200/.  The library is built by oracle.build() (oracle/__init__.py).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p


def build(force=False):
    return _build("segment_plane", force)


def lib():
    return load("segment_plane")


def segment_plane(pts, distance_threshold, ransac_n, seeds):
    """PointCloud::SegmentPlane (segmentation.cu:187-267) with one seed per iteration ->
    (plane float32[4], ascending inlier indices int32, best iteration or -1, fitness, inlier_rmse)"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    seeds = np.ascontiguousarray(seeds, np.int32).reshape(-1)
    plane, fr = np.zeros(4, np.float32), np.zeros(2, np.float32)
    idx = np.empty(max(len(pts), 1), np.int32)
    m, best = C.c_int(0), C.c_int(-1)
    rc = lib().orc_segment_plane(_p(pts), C.c_int(len(pts)), C.c_float(distance_threshold), C.c_int(ransac_n),
                                 C.c_int(len(seeds)), _p(seeds), _p(plane), _p(idx), C.byref(m), C.byref(best), _p(fr))
    assert rc == 0
    return plane, idx[:m.value].copy(), int(best.value), np.float32(fr[0]), np.float32(fr[1])


def ransac_keys(seed, n):
    keys = np.empty(n, np.int32)
    lib().orc_ransac_keys(C.c_int32(seed), C.c_int(n), _p(keys))
    return keys


def ransac_samples(n, seeds):
    """-> [T, 3] int32: d_cards[0..2] after each iteration's stable sort"""
    seeds = np.ascontiguousarray(seeds, np.int32).reshape(-1)
    out = np.empty((len(seeds), 3), np.int32)
    lib().orc_ransac_samples(C.c_int(n), C.c_int(len(seeds)), _p(seeds), _p(out))
    return out
