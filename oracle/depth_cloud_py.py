"""ctypes loader for the CreateFromDepthImage / CreateFromRGBDImage restatement (oracle/depth_cloud.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/, never by the product package cupoch_b200/.  The
library is built by oracle.build("depth_cloud") (oracle/__init__.py's recipe).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

_lib = None


def build(force=False):
    return _build("depth_cloud", force)


def lib():
    global _lib
    if _lib is None:
        _lib = load("depth_cloud")
        _lib.orc_depth_to_points.restype = C.c_longlong
        _lib.orc_depth_cloud_pose.restype = C.c_int
    return _lib


def _f(a, n):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(n))


def pose(E):
    """rows 0..2 of extrinsic^-1 (float64 Gauss-Jordan, rounded to float32), or None for a singular extrinsic"""
    P = np.empty(12, np.float32)
    return P.reshape(3, 4) if lib().orc_depth_cloud_pose(_p(_f(E, 16)), _p(P)) else None


def depth_to_points(depth, K, E=np.eye(4), depth_scale=1000.0, depth_trunc=1000.0, stride=1, color=None, depth_cutoff=-1.0,
                    compute_normals=False, project_valid_depth_only=True):
    """depth: [h, w] uint16 or float32; color: None, uint8 [h, w, 3] or float32 [h, w].  -> (points, normals or None,
    colors or None), [rows, 3] float32"""
    d = np.ascontiguousarray(depth)
    assert d.ndim == 2 and d.dtype in (np.uint16, np.float32)
    h, w = d.shape
    ct = 0
    c = None
    if color is not None:
        c = np.ascontiguousarray(color)
        ct = 1 if c.dtype == np.uint8 else 2
        assert c.shape[:2] == d.shape and (ct == 2) == (c.dtype == np.float32 and c.ndim == 2)
    K = np.asarray(K, np.float32).reshape(3, 3)
    K4 = np.float32([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    args = (_p(d), C.c_int(w), C.c_int(h), C.c_int(d.dtype.itemsize), C.c_int(int(depth_scale)), C.c_int(int(depth_trunc)),
            C.c_int(stride), _p(c), C.c_int(ct), _p(K4), _p(_f(E, 16)), C.c_float(depth_cutoff), C.c_int(int(bool(compute_normals))),
            C.c_int(int(bool(project_valid_depth_only))))
    L = lib()
    m = L.orc_depth_to_points(*args, None, None, None)
    if m < 0:
        raise ValueError("the extrinsic is not invertible")
    pts, nrm, col = (np.empty((max(m, 1), 3), np.float32) for _ in range(3))
    L.orc_depth_to_points(*args, _p(pts), _p(nrm), _p(col))
    return pts[:m], (nrm[:m] if compute_normals else None), (col[:m] if ct else None)
