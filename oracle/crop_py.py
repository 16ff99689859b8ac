"""ctypes loader for the bounding-box selection and point-cloud cleanup restatement (oracle/crop.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --crop, never by the product package
cupoch_b200/.  The library is built by oracle.build("crop") (oracle/__init__.py's recipe).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p


def build(force=False):
    return _build("crop", force)


def lib():
    return load("crop")


def _pts(pts):
    return np.ascontiguousarray(pts, np.float32).reshape(-1, 3)


def _f3(v):
    return np.ascontiguousarray(v, np.float32).reshape(-1)


def aabb_indices(pts, min_bound, max_bound):
    """ascending int32 indices of the points inside [min_bound, max_bound] (inclusive; NaN coordinates are kept)"""
    pts = _pts(pts)
    keep = np.zeros(len(pts), np.uint8)
    lo, hi = _f3(min_bound), _f3(max_bound)
    lib().orc_crop_aabb(_p(pts), C.c_int(len(pts)), _p(lo), _p(hi), _p(keep))
    return np.flatnonzero(keep).astype(np.int32)


def pass_through_indices(pts, axis, lo, hi):
    """PassThroughFilter's kept rows: the AABB test with [lo, hi] on `axis` and -inf / +inf on the other axes"""
    mn = np.full(3, -np.inf, np.float32)
    mx = np.full(3, np.inf, np.float32)
    mn[axis], mx[axis] = lo, hi
    return aabb_indices(pts, mn, mx)


def obb_indices(pts, box_points):
    """ascending int32 indices of the points the six determinant plane tests over box_points [8, 3] keep"""
    pts = _pts(pts)
    keep = np.zeros(len(pts), np.uint8)
    box = _f3(box_points)
    assert box.size == 24
    lib().orc_crop_obb(_p(pts), C.c_int(len(pts)), _p(box), _p(keep))
    return np.flatnonzero(keep).astype(np.int32)


def finite_indices(pts, remove_nan=True, remove_infinite=True):
    pts = _pts(pts)
    keep = np.zeros(len(pts), np.uint8)
    lib().orc_crop_finite(_p(pts), C.c_int(len(pts)), C.c_int(int(remove_nan)), C.c_int(int(remove_infinite)), _p(keep))
    return np.flatnonzero(keep).astype(np.int32)


def obb_create(pts):
    """OrientedBoundingBox::CreateFromPoints -> (center [3], R [3, 3] row-major, extent [3]), float32"""
    pts = _pts(pts)
    c, R, e = np.zeros(3, np.float32), np.zeros(9, np.float32), np.zeros(3, np.float32)
    lib().orc_obb_create(_p(pts), C.c_int(len(pts)), _p(c), _p(R), _p(e))
    return c, R.reshape(3, 3), e


def obb_box_points(center, R, extent):
    """OrientedBoundingBox::GetBoxPoints (boundingvolume.cu:180-194) in float32: axis_k = R[:, k] * (extent[k] / 2),
    corners center -+ x -+ y -+ z evaluated left to right"""
    c = np.asarray(center, np.float32)
    R = np.asarray(R, np.float32).reshape(3, 3)
    h = np.asarray(extent, np.float32) / np.float32(2)
    x, y, z = R[:, 0] * h[0], R[:, 1] * h[1], R[:, 2] * h[2]
    return np.stack([c - x - y - z, c + x - y - z, c - x + y - z, c - x - y + z,
                     c + x + y + z, c - x + y + z, c + x - y + z, c + x + y - z]).astype(np.float32)


def uniform_rows(n, every_k):
    """the rows UniformDownSample keeps: 0, k, 2k, ... (n // k of them); None for k < 1"""
    rows = np.zeros(max(n // max(int(every_k), 1), 1), np.int32)
    m = lib().orc_uniform_down_sample(C.c_int(n), C.c_int(int(every_k)), _p(rows))
    return None if m < 0 else rows[:m]


def normalize_normals(nrm):
    out = np.array(nrm, np.float32, copy=True).reshape(-1, 3)
    lib().orc_normalize_normals(_p(out), C.c_int(len(out)))
    return out


def orient_normals(nrm, reference):
    out = np.array(nrm, np.float32, copy=True).reshape(-1, 3)
    lib().orc_orient_normals(_p(out), C.c_int(len(out)), _p(_f3(reference)))
    return out
