"""ctypes loader for the TriangleMesh edge list / filter / area / sampling restatement (oracle/mesh_ops.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/, never by the product package cupoch_b200/.  The
library is built by oracle.build("mesh_ops").  Arrays are numpy; errors raise ValueError.
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

SHARPEN, SIMPLE, LAPLACIAN, TAUBIN = 0, 1, 2, 3
MAX_SAMPLES = 2 ** 30 - 1


def build(force=False):
    return _build("mesh_ops", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("mesh_ops")
        for f in ("orc_mesh_edge_list", "orc_mesh_filter", "orc_mesh_surface_area", "orc_mesh_sample"):
            getattr(_lib, f).restype = C.c_int
    return _lib


def _f3(a):
    return None if a is None else np.ascontiguousarray(a, np.float32).reshape(-1, 3)


def _check(rc):
    if rc == 1:
        raise ValueError("a vertex index is outside [0, n_vertices) or the edge list is not sorted")
    if rc == 2:
        raise ValueError("the surface area is not positive and finite")
    if rc:
        raise ValueError("bad argument")


def edge_list(triangles, n_vertices):
    """ComputeEdgeList -> [n, 2] int32, sorted and unique"""
    t = np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
    out = np.empty((max(6 * len(t), 1), 2), np.int32)
    n = C.c_longlong(0)
    _check(lib().orc_mesh_edge_list(_p(t), C.c_longlong(len(t)), C.c_longlong(n_vertices), _p(out), C.byref(n)))
    return out[:n.value]


def filter_mesh(kind, iterations, edges, vertices, normals=None, colors=None, mask=7, c0=1.0, c1=0.0):
    """one of the four filters -> (vertices, normals or None, colours or None); attributes outside mask are copied"""
    e = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
    v, n, c = _f3(vertices), _f3(normals), _f3(colors)
    outs = [None if a is None else np.empty_like(a) for a in (v, n, c)]
    _check(lib().orc_mesh_filter(C.c_int(kind), C.c_int(iterations), C.c_float(c0), C.c_float(c1), _p(e), C.c_longlong(len(e)),
                                 C.c_longlong(len(v)), _p(v), _p(n), _p(c), C.c_int(mask), *[_p(o) for o in outs]))
    return tuple(outs)


def sharpen(edges, vertices, normals=None, colors=None, iterations=1, strength=1.0, mask=7):
    return filter_mesh(SHARPEN, iterations, edges, vertices, normals, colors, mask, strength)


def smooth_simple(edges, vertices, normals=None, colors=None, iterations=1, mask=7):
    return filter_mesh(SIMPLE, iterations, edges, vertices, normals, colors, mask)


def smooth_laplacian(edges, vertices, normals=None, colors=None, iterations=1, lambda_=0.5, mask=7):
    return filter_mesh(LAPLACIAN, iterations, edges, vertices, normals, colors, mask, lambda_)


def smooth_taubin(edges, vertices, normals=None, colors=None, iterations=1, lambda_=0.5, mu=-0.53, mask=7):
    return filter_mesh(TAUBIN, iterations, edges, vertices, normals, colors, mask, lambda_, mu)


def surface_area(vertices, triangles):
    """GetSurfaceArea -> (total as np.float32, per-triangle areas float32)"""
    v, t = _f3(vertices), np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
    areas, total = np.empty(max(len(t), 1), np.float32), C.c_float(0)
    _check(lib().orc_mesh_surface_area(_p(v), C.c_longlong(len(v)), _p(t), C.c_longlong(len(t)), _p(areas), C.byref(total)))
    return np.float32(total.value), areas[:len(t)]


def sample_points_uniformly(vertices, triangles, n, vertex_normals=None, triangle_normals=None, vertex_colors=None, normals=True):
    """SamplePointsUniformly -> (points, normals or None, colours or None, boundaries [nt + 1] uint32).  Normals are
    written when normals is True and triangle_normals or vertex_normals is given (triangle normals first)."""
    v, t = _f3(vertices), np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
    vn, tn, vc = _f3(vertex_normals), _f3(triangle_normals), _f3(vertex_colors)
    n = int(n)
    if n <= 0 or n > MAX_SAMPLES or len(t) == 0:
        raise ValueError("bad argument")
    pts = np.empty((n, 3), np.float32)
    nrm = np.empty((n, 3), np.float32) if normals and (vn is not None or tn is not None) else None
    col = np.empty((n, 3), np.float32) if vc is not None else None
    bnd = np.empty(len(t) + 1, np.uint32)
    _check(lib().orc_mesh_sample(_p(v), C.c_longlong(len(v)), _p(t), C.c_longlong(len(t)), _p(vn), _p(tn), _p(vc), C.c_longlong(n),
                                 _p(pts), _p(nrm), _p(col), _p(bnd)))
    return pts, nrm, col, bnd
