"""ctypes loader for the FarthestPointDownSample restatement (oracle/fps.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --fps, never by the product package
cupoch_b200/.  The library is built by oracle.build() (oracle/__init__.py).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p


def build(force=False):
    return _build("fps", force)


def lib():
    return load("fps")


def farthest_point_down_sample(pts, num_samples):
    """-> (indices [num_samples] int32, final running distances [n] float32); the loop runs for any num_samples
    (DESIGN.md arithmetic contract, smallest index among equal distances).  No points: nothing to pick, both empty."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    n, k = len(pts), int(num_samples)
    if n == 0:
        return np.empty(0, np.int32), np.empty(0, np.float32)
    idx = np.empty(k, np.int32)
    dist = np.empty(n, np.float32)
    lib().orc_farthest_point_down_sample(_p(pts), C.c_int(n), C.c_long(k), _p(idx), _p(dist))
    return idx, dist
