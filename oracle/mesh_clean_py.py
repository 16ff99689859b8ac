"""ctypes loader for the mesh cleanup and self-intersection restatement (oracle/mesh_clean.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/, never by the product package cupoch_b200/.  The
library is built by oracle.build("mesh_clean").  Arrays are numpy; a bad vertex index raises ValueError.
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

ALL_PAIRS, SWEEP = 0, 1
_LL = C.c_longlong


def build(force=False):
    return _build("mesh_clean", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("mesh_clean")
        for f in ("orc_remove_duplicated_vertices", "orc_remove_duplicated_triangles", "orc_remove_unreferenced_vertices",
                  "orc_remove_degenerate_triangles", "orc_append_triangles", "orc_tritri", "orc_self_intersections"):
            getattr(_lib, f).restype = C.c_int
    return _lib


def _f(a):
    return None if a is None else np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, 3))


def _i(a):
    return np.ascontiguousarray(np.asarray(a, np.int32).reshape(-1, 3))


def _check(rc):
    if rc == 1:
        raise ValueError("a vertex index is outside [0, n_vertices)")


def _vertex_op(fn, vertices, triangles, normals, colors):
    v, t, vn, vc = _f(vertices), _i(triangles), _f(normals), _f(colors)
    ov, ot = np.empty_like(v), np.empty_like(t)
    on = None if vn is None else np.empty_like(v)
    oc = None if vc is None else np.empty_like(v)
    k = _LL(0)
    _check(fn(_p(v), _p(vn), _p(vc), _LL(len(v)), _p(t), _LL(len(t)), _p(ov), _p(on), _p(oc), _p(ot), C.byref(k)))
    k = k.value
    return ov[:k].copy(), ot, None if on is None else on[:k].copy(), None if oc is None else oc[:k].copy()


def _triangle_op(fn, triangles, n_vertices, triangle_normals):
    t, tn = _i(triangles), _f(triangle_normals)
    ot = np.empty_like(t)
    otn = None if tn is None else np.empty_like(tn)
    k = _LL(0)
    _check(fn(_p(t), _p(tn), _LL(len(t)), _LL(n_vertices), _p(ot), _p(otn), C.byref(k)))
    k = k.value
    return ot[:k].copy(), None if otn is None else otn[:k].copy()


def remove_duplicated_vertices(vertices, triangles, normals=None, colors=None):
    """-> (vertices, triangles, normals, colours): distinct positions in lexicographic order, lowest index survives"""
    return _vertex_op(lib().orc_remove_duplicated_vertices, vertices, triangles, normals, colors)


def remove_unreferenced_vertices(vertices, triangles, normals=None, colors=None):
    """-> (vertices, triangles, normals, colours): the referenced vertices in order"""
    return _vertex_op(lib().orc_remove_unreferenced_vertices, vertices, triangles, normals, colors)


def remove_duplicated_triangles(triangles, n_vertices, triangle_normals=None):
    """-> (triangles, triangle normals): aligned, sorted, first of each run"""
    return _triangle_op(lib().orc_remove_duplicated_triangles, triangles, n_vertices, triangle_normals)


def remove_degenerate_triangles(triangles, n_vertices, triangle_normals=None):
    """-> (triangles, triangle normals): those with three distinct indices, in order"""
    return _triangle_op(lib().orc_remove_degenerate_triangles, triangles, n_vertices, triangle_normals)


def append_triangles(tri_a, nv_a, tri_b, nv_b):
    a, b = _i(tri_a), _i(tri_b)
    out = np.empty((len(a) + len(b), 3), np.int32)
    _check(lib().orc_append_triangles(_p(a), _LL(len(a)), _LL(nv_a), _p(b), _LL(len(b)), _LL(nv_b), _p(out)))
    return out


def tritri(p, q):
    """TriangleTriangle3d on two triangles given as 3 x 3 float32 arrays"""
    return bool(lib().orc_tritri(_p(np.ascontiguousarray(np.asarray(p, np.float32).reshape(9))),
                                 _p(np.ascontiguousarray(np.asarray(q, np.float32).reshape(9)))))


def self_intersections(vertices, triangles, mode=SWEEP, filtered=True):
    """-> pairs [n, 2] int32 in ascending (i, j) order.  ALL_PAIRS is the reference's loop (filtered adds the finite and
    box-overlap conditions); SWEEP is always filtered."""
    v, t = _f(vertices), _i(triangles)
    cap = 1 << 12
    while True:
        out = np.empty((cap, 2), np.int32)
        n = _LL(0)
        rc = lib().orc_self_intersections(_p(v), _LL(len(v)), _p(t), _LL(len(t)), C.c_int(mode), C.c_int(int(bool(filtered))), _p(out),
                                          _LL(cap), C.byref(n))
        _check(rc)
        if rc == 0:
            return out[:n.value].copy()
        cap = n.value
