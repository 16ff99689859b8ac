"""ctypes loader for the ComputeSHOTFeature restatement (oracle/shot.c, compiled together with oracle/oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --shot, never by the product package
cupoch_b200/.  The library is built by oracle.build() (oracle/__init__.py).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

DIM = 352


def build(force=False):
    return _build("shot", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("shot")
        _lib.orc_compute_shot_feature.restype = C.c_int
        _lib.orc_shot_neighbours.restype = C.c_int
        _lib.orc_shot_from_neighbours.restype = None
    return _lib


def _search(search_param):
    """(knn, search_radius, max_nn) from a KDTreeSearchParam-like object or a tuple"""
    if isinstance(search_param, tuple):
        return search_param
    if hasattr(search_param, "knn"):
        return int(search_param.knn), 0.0, 0
    return 0, float(search_param.radius), int(search_param.max_nn)


def compute_shot_feature(pts, nrm, radius, knn=0, search_radius=0.0, max_nn=0):
    """-> [n, 352] float32.  knn > 0: KNN(knn) search, else Radius(search_radius, max_nn)."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    nrm = np.ascontiguousarray(nrm, np.float32).reshape(-1, 3)
    n = len(pts)
    out = np.zeros((max(n, 1), DIM), np.float32)
    rc = lib().orc_compute_shot_feature(_p(pts), _p(nrm), C.c_int(n), C.c_float(radius), C.c_int(knn),
                                        C.c_float(search_radius), C.c_int(max_nn), _p(out))
    if rc < 0:
        raise ValueError("knn must be <= 100 and max_nn must lie in [0, 256]")
    return out[:n]


def neighbours(pts, knn=0, search_radius=0.0, max_nn=0):
    """the lists the descriptor reads -> (idx [n, k] int32, -1 = empty slot; d2 [n, k] float32), ascending (d2, index)"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    n = len(pts)
    k = knn if knn > 0 else max_nn
    idx = np.full((max(n, 1), max(k, 1)), -1, np.int32)
    d2 = np.full((max(n, 1), max(k, 1)), np.inf, np.float32)
    rc = lib().orc_shot_neighbours(_p(pts), C.c_int(n), C.c_int(knn), C.c_float(search_radius), C.c_int(max_nn),
                                   _p(idx), _p(d2))
    if rc < 0:
        raise ValueError("knn must be <= 100 and max_nn must lie in [0, 256]")
    return idx[:n, :k], d2[:n, :k]


def shot_from_neighbours(pts, nrm, idx, d2, radius):
    """the descriptor over given tables [n, k]"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    nrm = np.ascontiguousarray(nrm, np.float32).reshape(-1, 3)
    idx = np.ascontiguousarray(idx, np.int32)
    d2 = np.ascontiguousarray(d2, np.float32)
    n, k = idx.shape
    out = np.zeros((max(n, 1), DIM), np.float32)
    if n and k:
        lib().orc_shot_from_neighbours(_p(pts), _p(nrm), C.c_int(n), _p(idx), _p(d2), C.c_int(k), C.c_float(radius),
                                       _p(out))
    return out[:n]
