"""ctypes loader for the VoxelGrid operations restatement (oracle/voxelgrid_ops.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --voxelgrid, never by the product
package cupoch_b200/.  The library is built by oracle.build("voxelgrid_ops") (oracle/__init__.py's recipe).  A grid is
(keys [n, 3] int32, colors [n, 3] float32); the element-wise operations (paint, select, the OccupancyGrid point
formula) are restated here in numpy float32, which rounds each operation as the kernels do.
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p


def build(force=False):
    return _build("voxelgrid_ops", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("voxelgrid_ops")
        _lib.orc_vg_dense_counts.restype = C.c_int
        _lib.orc_vg_merge.restype = C.c_int64
        for f in ("orc_vg_dense", "orc_vg_included", "orc_vg_carve"):
            getattr(_lib, f).restype = None
    return _lib


def _f(a, n):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(n))


def _k(keys):
    return np.ascontiguousarray(np.asarray(keys, np.int32).reshape(-1, 3))


def dense_counts(vs, w, h, d):
    """-> (nw, nh, nd), or None when CreateDense rejects the arguments"""
    cnt = np.zeros(3, np.int64)
    if lib().orc_vg_dense_counts(C.c_float(vs), C.c_float(w), C.c_float(h), C.c_float(d), _p(cnt)):
        return None
    return tuple(int(c) for c in cnt)


def create_dense(vs, w, h, d):
    cnt = np.asarray(dense_counts(vs, w, h, d), np.int64)
    m = int(np.prod(cnt))
    keys, cols = np.empty((m, 3), np.int32), np.empty((m, 3), np.float32)
    if m:
        lib().orc_vg_dense(_p(cnt), _p(keys), _p(cols))
    return keys, cols


def check_if_included(keys, vs, origin, queries):
    keys, q = _k(keys), np.ascontiguousarray(np.asarray(queries, np.float32).reshape(-1, 3))
    out = np.zeros(max(len(q), 1), np.uint8)
    lib().orc_vg_included(_p(keys), C.c_int64(len(keys)), C.c_float(vs), _p(_f(origin, 3)), _p(q), C.c_int64(len(q)), _p(out))
    return out[:len(q)].astype(bool)


def carve_keep(keys, vs, origin, image, intrinsic, extrinsic, keep_outside):
    """per voxel: survives the carve.  image: a numpy (h, w[, c]) array; only 1-channel float32 is sampled."""
    keys, img = _k(keys), np.ascontiguousarray(image)
    h, w = img.shape[:2]
    sampled = int(img.dtype == np.float32 and (img.ndim == 2 or img.shape[2] == 1))
    keep = np.zeros(max(len(keys), 1), np.uint8)
    lib().orc_vg_carve(_p(keys), C.c_int64(len(keys)), C.c_float(vs), _p(_f(origin, 3)), _p(img) if sampled else None, C.c_int(w),
                       C.c_int(h), C.c_int(sampled), _p(_f(intrinsic, 9)), _p(_f(extrinsic, 16)), C.c_int(int(bool(keep_outside))),
                       _p(keep))
    return keep[:len(keys)].astype(bool)


def carve(keys, colors, vs, origin, image, intrinsic, extrinsic, keep_outside):
    k = carve_keep(keys, vs, origin, image, intrinsic, extrinsic, keep_outside)
    return _k(keys)[k], np.asarray(colors, np.float32).reshape(-1, 3)[k]


def merge(keys_a, colors_a, keys_b, colors_b, average=True):
    """+= (average) or AddVoxels (first of each run)"""
    keys = np.ascontiguousarray(np.concatenate([_k(keys_a), _k(keys_b)]))
    cols = np.ascontiguousarray(np.concatenate([np.asarray(colors_a, np.float32).reshape(-1, 3),
                                                np.asarray(colors_b, np.float32).reshape(-1, 3)]))
    n = len(keys)
    ok, oc = np.empty((max(n, 1), 3), np.int32), np.empty((max(n, 1), 3), np.float32)
    m = lib().orc_vg_merge(_p(keys), _p(cols), C.c_int64(n), C.c_int(int(bool(average))), _p(ok), _p(oc))
    return ok[:m].copy(), oc[:m].copy()


def paint(colors, indices, color):
    c = np.array(colors, np.float32).reshape(-1, 3)
    c[np.arange(len(c)) if indices is None else np.asarray(indices, np.int64)] = np.asarray(color, np.float32)
    return c


def select(keys, colors, indices, invert=False):
    idx = np.asarray(indices, np.int64).reshape(-1)
    if invert:
        idx = np.setdiff1d(np.arange(len(keys)), idx)
    return _k(keys)[idx], np.asarray(colors, np.float32).reshape(-1, 3)[idx]


def occ_points(cells, res, vs, origin):
    """compute_points_from_occvoxels_functor: (cell + (float)(-(res / 2) + 0.5)) * vs + origin, each step in float32"""
    c = np.float32(-(res // 2) + 0.5)
    return ((np.asarray(cells, np.int32).astype(np.float32) + c) * np.float32(vs) + _f(origin, 3)).astype(np.float32)


def occ_voxel_origin(res, vs, origin):
    return (_f(origin, 3) - np.float32(res // 2) * np.float32(vs)).astype(np.float32)
