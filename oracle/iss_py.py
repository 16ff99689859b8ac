"""ctypes loader for the ComputeISSKeypoints restatement (oracle/iss.c, compiled together with oracle/oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --iss, never by the product package
cupoch_b200/.  The library is built by oracle.build() (oracle/__init__.py).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p


def build(force=False):
    return _build("iss", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("iss")
        _lib.orc_iss_keypoints.restype = C.c_int
    return _lib


def iss_keypoints(pts, salient_radius=0.0, non_max_radius=0.0, gamma_21=0.975, gamma_32=0.975, min_neighbors=5,
                  max_neighbors=100):
    """-> (mask [n] bool, saliency [n] float32, radii used float32[2]); both radii are replaced by 6 and 4 times the
    resolution when either is 0."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    n = len(pts)
    mask = np.zeros(max(n, 1), np.uint8)
    sal = np.zeros(max(n, 1), np.float32)
    radii = np.zeros(2, np.float32)
    rc = lib().orc_iss_keypoints(_p(pts), C.c_int(n), C.c_float(salient_radius), C.c_float(non_max_radius),
                                 C.c_float(gamma_21), C.c_float(gamma_32), C.c_int(min_neighbors), C.c_int(max_neighbors),
                                 _p(mask), _p(sal), _p(radii))
    if rc < 0:
        raise ValueError("max_neighbors must lie in [0, 256]")
    return mask[:n].astype(bool), sal[:n], radii
