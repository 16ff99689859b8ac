"""ctypes loader for the collision restatement (oracle/collision.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --collision, never by the product
package cupoch_b200/.  The library is built by oracle.build("collision") (oracle/__init__.py's recipe).

Operands are plain dicts: a grid is {"keys": [n, 3] int32, "ids": [n] int32 ascending, "vs": float, "origin": [3]},
primitives are a PRIM_DTYPE array.  compute(a, b, margin) -> [m, 2] int32 pairs (target index, query index).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

BOX, SPHERE, CAPSULE, CYLINDER = 1, 2, 3, 4
PRIM_DTYPE = np.dtype([("type", np.int32), ("transform", np.float32, (16,)), ("lengths", np.float32, (3,)),
                       ("radius", np.float32), ("height", np.float32)])


def build(force=False):
    return _build("collision", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("collision")
        _lib.orc_coll_prim_elem.restype = C.c_int
        _lib.orc_coll_elem_elem.restype = C.c_int
        for f in ("orc_coll_grid_grid", "orc_coll_prim_grid"):
            getattr(_lib, f).restype = None
    return _lib


def prim(type, transform=None, lengths=(0, 0, 0), radius=0.0, height=0.0):
    """one primitive record (transform row-major 4x4, identity by default)"""
    p = np.zeros((), PRIM_DTYPE)
    p["type"] = type
    p["transform"] = np.asarray(np.eye(4) if transform is None else transform, np.float32).reshape(16)
    p["lengths"] = np.asarray(lengths, np.float32).reshape(3)
    p["radius"], p["height"] = radius, height
    return p


def prims(records):
    return np.ascontiguousarray(np.array([np.asarray(r, PRIM_DTYPE) for r in records], PRIM_DTYPE).reshape(-1))


def voxel_grid(keys, vs, origin):
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, 3)
    return {"keys": keys, "ids": np.arange(len(keys), dtype=np.int32), "vs": float(np.float32(vs)),
            "origin": np.asarray(origin, np.float32).reshape(3)}


def occupied(prob, lo, hi, thres):
    """the occupied cells of a dense [res, res, res] log-odds grid inside the bound box [lo, hi] (grid indices):
    !isnan(p) && p > thres, ascending linear index -> (cells [m, 3] int32, linear [m] int32)"""
    prob = np.asarray(prob, np.float32)
    r = prob.shape[0]
    occ = ~np.isnan(prob) & (prob > np.float32(thres))
    box = np.zeros_like(occ)
    lo, hi = np.asarray(lo, int), np.asarray(hi, int)
    if np.all(hi >= lo):
        box[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = True
    lin = np.flatnonzero((occ & box).reshape(-1)).astype(np.int32)
    cells = np.stack([lin // (r * r), (lin // r) % r, lin % r], 1).astype(np.int32)
    return cells, lin


def occupancy_grid(prob, lo, hi, thres, vs, origin):
    """an OccupancyGrid operand: cell (x, y, z) has key (x, y, z) - res // 2 and index x * res^2 + y * res + z"""
    cells, lin = occupied(prob, lo, hi, thres)
    half = np.asarray(prob).shape[0] // 2
    return {"keys": np.ascontiguousarray(cells - half, np.int32), "ids": lin, "vs": float(np.float32(vs)),
            "origin": np.asarray(origin, np.float32).reshape(3)}


def _f3(v):
    return np.ascontiguousarray(np.asarray(v, np.float32).reshape(3))


def best(a, b, margin):
    """per query element of b: the smallest colliding index of a, or -1"""
    m = C.c_float(float(np.float32(margin)))
    if isinstance(b, np.ndarray):  # primitive query
        g = a
        out = np.empty(max(len(b), 1), np.int32)
        lib().orc_coll_prim_grid(_p(b), C.c_int64(len(b)), _p(g["keys"]), _p(g["ids"]), C.c_int64(len(g["keys"])), C.c_float(g["vs"]),
                                 _p(_f3(g["origin"])), m, C.c_int(0), _p(out))
        return out[:len(b)]
    nq = len(b["keys"])
    out = np.empty(max(nq, 1), np.int32)
    if isinstance(a, np.ndarray):  # primitive target
        lib().orc_coll_prim_grid(_p(a), C.c_int64(len(a)), _p(b["keys"]), _p(b["ids"]), C.c_int64(nq), C.c_float(b["vs"]),
                                 _p(_f3(b["origin"])), m, C.c_int(1), _p(out))
    else:
        lib().orc_coll_grid_grid(_p(a["keys"]), _p(a["ids"]), C.c_int64(len(a["keys"])), C.c_float(a["vs"]), _p(_f3(a["origin"])),
                                 _p(b["keys"]), C.c_int64(nq), C.c_float(b["vs"]), _p(_f3(b["origin"])), m, _p(out))
    return out[:nq]


def compute(a, b, margin=0.0):
    """ComputeIntersection(a, b, margin) -> [m, 2] int32 (target index, query index), ascending query order"""
    bst = best(a, b, margin)
    qid = np.arange(len(bst), dtype=np.int32) if isinstance(b, np.ndarray) else b["ids"]
    hit = bst >= 0
    return np.ascontiguousarray(np.stack([bst[hit], np.asarray(qid)[hit]], 1).astype(np.int32).reshape(-1, 2))


def prim_elem(p, key, vs, origin, margin=0.0):
    """one primitive against one grid element"""
    p = np.ascontiguousarray(np.asarray(p, PRIM_DTYPE).reshape(1))
    k = np.ascontiguousarray(key, np.int32).reshape(3)
    return bool(lib().orc_coll_prim_elem(_p(p), _p(k), C.c_float(vs), _p(_f3(origin)), C.c_float(margin)))


def elem_elem(kt, tvs, to, kq, qvs, qo, margin=0.0):
    kt, kq = np.ascontiguousarray(kt, np.int32).reshape(3), np.ascontiguousarray(kq, np.int32).reshape(3)
    return bool(lib().orc_coll_elem_elem(_p(kt), C.c_float(tvs), _p(_f3(to)), _p(kq), C.c_float(qvs), _p(_f3(qo)), C.c_float(margin)))
