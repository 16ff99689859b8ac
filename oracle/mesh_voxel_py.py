"""ctypes loader for the mesh voxelisation restatement (oracle/mesh_voxel.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/, never by the product package cupoch_b200/.  The
library is built by oracle.build("mesh_voxel").  Arrays are numpy; errors raise ValueError.
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

CELL_MAJOR, TRIANGLE_MAJOR = 0, 1


def build(force=False):
    return _build("mesh_voxel", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("mesh_voxel")
        for f in ("orc_mesh_voxel", "orc_mesh_voxel_counts", "orc_tri_box"):
            getattr(_lib, f).restype = C.c_int
    return _lib


def _f3(a):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(3))


def counts(voxel_size, min_bound, max_bound):
    """-> (n_x, n_y, n_z), the count rule; ValueError when the arguments are rejected"""
    cnt = np.zeros(3, np.int64)
    if lib().orc_mesh_voxel_counts(C.c_float(voxel_size), _p(_f3(min_bound)), _p(_f3(max_bound)), _p(cnt)):
        raise ValueError("bad voxel size, bounds or count")
    return tuple(int(c) for c in cnt)


def tri_box(centre, half, a, b, c):
    """the float32 triangle/box overlap test on one box"""
    return bool(lib().orc_tri_box(_p(_f3(centre)), C.c_float(half), _p(_f3(a)), _p(_f3(b)), _p(_f3(c))))


def voxelize(vertices, triangles, voxel_size, min_bound, max_bound, mode=TRIANGLE_MAJOR, corner=False):
    """CreateFromTriangleMeshWithinBounds -> keys [m, 3] int32, unique and in lexicographic order.  corner: test the box
    centred at k * vs + min_bound (the reference's rule) instead of the cell centre."""
    v = np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3))
    t = np.ascontiguousarray(np.asarray(triangles, np.int32).reshape(-1, 3))
    cap = 1 << 16
    while True:
        out = np.empty((cap, 3), np.int32)
        n = C.c_longlong(0)
        rc = lib().orc_mesh_voxel(_p(v), C.c_longlong(len(v)), _p(t), C.c_longlong(len(t)), C.c_float(voxel_size),
                                  _p(_f3(min_bound)), _p(_f3(max_bound)), C.c_int(mode), C.c_int(int(bool(corner))), _p(out),
                                  C.c_longlong(cap), C.byref(n))
        if rc == 1:
            raise ValueError("a vertex index is outside [0, n_vertices)")
        if rc == 2:
            raise ValueError("bad voxel size, bounds or count")
        if rc == 0:
            return out[:n.value].copy()
        cap = n.value
