"""ctypes loader for the DistanceTransform restatement (oracle/edt.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --edt, never by the product package
cupoch_b200/.  The library is compiled on first use with oracle/Makefile's flags into oracle/_build/ (or a per-user
temporary directory when the tree is read-only).
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "edt.c")
CFLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wextra", "-Wno-unused-parameter",
          "-Wno-unknown-pragmas"]
NOT_SITE = 2  # DistanceVoxel::NotSite


def build(force=False):
    out_dir = os.path.join(_HERE, "_build")
    if not os.access(_HERE, os.W_OK) and not os.access(out_dir, os.W_OK):
        out_dir = os.path.join(tempfile.gettempdir(), "cphb_oracle_%d" % os.getuid())
    so = os.path.join(out_dir, "libedt.so")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(_SRC):
        os.makedirs(out_dir, exist_ok=True)
        cmd = [os.environ.get("CC", "gcc")] + CFLAGS + ["-shared", "-o", so, _SRC, "-lm"]
        # OpenMP only parallelises over lines (each line's result is computed alone): single-threaded if unavailable
        if subprocess.run(cmd[:1] + ["-fopenmp"] + cmd[1:], capture_output=True).returncode != 0:
            subprocess.check_call(cmd)
    return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_dt_voxel_size_ok.restype = C.c_int
        _lib.orc_dt_voxel_size_ok.argtypes = [C.c_float, C.c_float]
        for f in ("orc_dt_key_cells", "orc_dt_compute", "orc_dt_distance_index", "orc_dt_voxel_index"):
            getattr(_lib, f).restype = None
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f3(v):
    return np.ascontiguousarray(np.asarray(v, np.float32).reshape(3))


def voxel_size_ok(vs_dt, vs_vg):
    """|vs_dt - vs_vg| <= FLT_EPSILON in float32 (otherwise the reference logs and leaves the grid unchanged)"""
    return bool(lib().orc_dt_voxel_size_ok(float(np.float32(vs_dt)), float(np.float32(vs_vg))))


def key_cells(keys, vs, origin_vg, origin_dt, res):
    """VoxelGrid keys [n, 3] -> (grid cells [n, 3] int32, inside [n] bool)"""
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, 3)
    n = len(keys)
    cells = np.zeros((max(n, 1), 3), np.int32)
    inside = np.zeros(max(n, 1), np.uint8)
    lib().orc_dt_key_cells(_p(keys), C.c_int64(n), C.c_float(vs), _p(_f3(origin_vg)), _p(_f3(origin_dt)), C.c_int(res),
                           _p(cells), _p(inside))
    return cells[:n], inside[:n].astype(bool)


def compute(res, cells, voxel_size=1.0, with_distance=True):
    """ComputeEDT (with_distance) / ComputeVoronoiDiagram of grid cells [n, 3] on a fresh res^3 grid
    -> (nearest [res, res, res, 3] uint16, state [res, res, res] uint8, distance [res, res, res] float32)"""
    cells = np.ascontiguousarray(cells, np.int32).reshape(-1, 3)
    if not len(cells):
        cells = np.zeros((0, 3), np.int32)
    r = int(res)
    nearest = np.empty((r, r, r, 3), np.uint16)
    state = np.empty((r, r, r), np.uint8)
    dist = np.empty((r, r, r), np.float32)
    lib().orc_dt_compute(C.c_int(r), _p(cells) if len(cells) else None, C.c_int64(len(cells)), C.c_int(1 if with_distance else 0),
                         C.c_float(voxel_size), _p(nearest), _p(state), _p(dist))
    return nearest, state, dist


def compute_voxel_grid(res, voxel_size, origin, keys, vg_voxel_size, vg_origin, with_distance=True):
    """ComputeEDT / ComputeVoronoiDiagram(VoxelGrid) on a fresh grid; None when the voxel sizes differ (grid unchanged)"""
    if not voxel_size_ok(voxel_size, vg_voxel_size):
        return None
    cells, inside = key_cells(keys, voxel_size, vg_origin, origin, res)
    return compute(res, cells[inside], voxel_size, with_distance)


def occupied_cells(prob, thres):
    """CreateFromOccupancyGrid's sites: the cells of the dense log-odds array with !isnan(p) && p > thres"""
    prob = np.asarray(prob, np.float32)
    r = prob.shape[0]
    flat = np.flatnonzero(~np.isnan(prob.reshape(-1)) & (prob.reshape(-1) > np.float32(thres)))
    return np.stack([flat // (r * r), (flat // r) % r, flat % r], 1).astype(np.int32)


def default_grid(res):
    """a fresh grid: nearest (0,0,0), NotSite, distance 0"""
    r = int(res)
    return np.zeros((r, r, r, 3), np.uint16), np.full((r, r, r), NOT_SITE, np.uint8), np.zeros((r, r, r), np.float32)


def reconstruct(grid, res):
    """DenseGrid::Reconstruct (densegrid.inl:128-134): the linear prefix of the old cells, defaults after it"""
    out = default_grid(res)
    for o, a in zip(out, grid):
        fo, fa = o.reshape(o.shape[0] ** 3, -1), a.reshape(a.shape[0] ** 3, -1)
        m = min(len(fo), len(fa))
        fo[:m] = fa[:m]
    return out


def _index(fn, points, voxel_size, origin, res):
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    idx = np.empty(max(len(pts), 1), np.int64)
    getattr(lib(), fn)(_p(pts), C.c_int64(len(pts)), C.c_float(voxel_size), _p(_f3(origin)), C.c_int(res), _p(idx))
    return idx[:len(pts)]


def distance_index(points, voxel_size, origin, res):
    """the cell get_distance / get_distances read: linear index, or -1 outside the grid / NaN"""
    return _index("orc_dt_distance_index", points, voxel_size, origin, res)


def voxel_index(points, voxel_size, origin, res):
    """the cell get_voxel reads: linear index, or -1 outside the grid / NaN"""
    return _index("orc_dt_voxel_index", points, voxel_size, origin, res)


def get_distances(dist, points, voxel_size, origin):
    """GetDistances over an oracle distance grid: 0 outside the grid"""
    idx = distance_index(points, voxel_size, origin, dist.shape[0])
    return np.where(idx >= 0, dist.reshape(-1)[np.maximum(idx, 0)], np.float32(0)).astype(np.float32)
