"""ctypes loader for the UniformTSDFVolume restatement (oracle/tsdf.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/, never by the product package cupoch_b200/.  The
library is built by oracle.build("tsdf") (oracle/__init__.py's recipe).  Volume holds the kernel's planes on the host:
tw [N, 2] float32 (tsdf, weight) and col [planes, N] float32 (3 planes for RGB8, 1 for Gray32, none for NoColor).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

NO_COLOR, RGB8, GRAY32 = 0, 1, 2
PLANES = {NO_COLOR: 0, RGB8: 3, GRAY32: 1}


def build(force=False):
    return _build("tsdf", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("tsdf")
        for f in ("orc_tsdf_extract_points", "orc_tsdf_extract_voxels"):
            getattr(_lib, f).restype = C.c_longlong
        for f in ("orc_tsdf_depth_to_float", "orc_tsdf_intensity", "orc_tsdf_reset", "orc_tsdf_integrate", "orc_tsdf_raycast",
                  "orc_tsdf_pose"):
            getattr(_lib, f).restype = None
    return _lib


def _f(a, n):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(n))


def k4(K):
    """(fx, fy, cx, cy) of a 3x3 intrinsic matrix"""
    K = np.asarray(K, np.float32).reshape(3, 3)
    return np.float32([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])


def depth_to_float(depth, depth_scale=1000.0, depth_trunc=3.0):
    """ConvertDepthToFloatImage with the scale and truncation converted to int, as the reference's functor takes them"""
    d = np.ascontiguousarray(depth)
    out = np.empty(d.shape[:2], np.float32)
    lib().orc_tsdf_depth_to_float(_p(d), C.c_int(d.dtype.itemsize), C.c_longlong(out.size), C.c_int(int(depth_scale)),
                                  C.c_int(int(depth_trunc)), _p(out))
    return out


def intensity(color):
    """CreateFloatImage(WEIGHTED) of a 1- or 3-channel image"""
    c = np.ascontiguousarray(color)
    ch = 1 if c.ndim == 2 else c.shape[2]
    out = np.empty(c.shape[:2], np.float32)
    lib().orc_tsdf_intensity(_p(c), C.c_int(ch), C.c_int(c.dtype.itemsize), C.c_longlong(out.size), _p(out))
    return out


def pose(E):
    P = np.empty(12, np.float32)
    lib().orc_tsdf_pose(_p(_f(E, 16)), _p(P))
    return P.reshape(3, 4)


class Volume:
    def __init__(self, length, resolution, sdf_trunc, color_type=NO_COLOR, origin=(0.0, 0.0, 0.0)):
        self.length, self.res, self.trunc, self.ct = float(length), int(resolution), float(sdf_trunc), int(color_type)
        self.origin = _f(origin, 3)
        n = self.res ** 3
        self.tw = np.zeros((n, 2), np.float32)
        self.col = np.zeros((PLANES[self.ct], n), np.float32)
        self.reset()

    @property
    def voxel_length(self):
        return np.float32(self.length) / np.float32(self.res)

    def reset(self):
        lib().orc_tsdf_reset(_p(self.tw), _p(self.col), C.c_int(PLANES[self.ct]), C.c_longlong(self.res ** 3))

    def integrate(self, depth, color, K, E):
        """depth: float32 [h, w] metres; color: uint8 [h, w, 3] (RGB8), float32 [h, w] (Gray32) or None"""
        d = np.ascontiguousarray(depth, np.float32)
        h, w = d.shape
        c = None if color is None or self.ct == NO_COLOR else np.ascontiguousarray(color)
        lib().orc_tsdf_integrate(_p(self.tw), _p(self.col), C.c_float(self.length), C.c_int(self.res), C.c_float(self.trunc),
                                 C.c_int(self.ct), _p(self.origin), _p(d), _p(c), C.c_int(w), C.c_int(h), _p(k4(K)), _p(_f(E, 16)))

    def extract_point_cloud(self):
        L = lib()
        args = (_p(self.tw), _p(self.col), C.c_float(self.length), C.c_int(self.res), C.c_float(self.trunc), C.c_int(self.ct),
                _p(self.origin))
        m = L.orc_tsdf_extract_points(*args, None, None, None, C.c_longlong(0))
        pts, nrm, col = (np.empty((max(m, 1), 3), np.float32) for _ in range(3))
        L.orc_tsdf_extract_points(*args, _p(pts), _p(nrm), _p(col), C.c_longlong(m))
        return pts[:m], nrm[:m], (col[:m] if self.ct != NO_COLOR else None)

    def _voxels(self):
        L = lib()
        args = (_p(self.tw), C.c_float(self.length), C.c_int(self.res), _p(self.origin))
        m = L.orc_tsdf_extract_voxels(*args, None, None, None, C.c_longlong(0))
        keys, pts, col = np.empty((max(m, 1), 3), np.int32), np.empty((max(m, 1), 3), np.float32), np.empty((max(m, 1), 3), np.float32)
        L.orc_tsdf_extract_voxels(*args, _p(keys), _p(pts), _p(col), C.c_longlong(m))
        return keys[:m], pts[:m], col[:m]

    def extract_voxel_point_cloud(self):
        _, pts, col = self._voxels()
        return pts, col

    def extract_voxel_grid(self):
        """-> (keys, colors, voxel_size, grid origin = origin - (res / 2) * vl)"""
        keys, _, col = self._voxels()
        vl = self.voxel_length
        return keys, col, vl, (self.origin - np.float32(self.res // 2) * vl).astype(np.float32)

    def raycast(self, K, E, w, h, sdf_trunc, project_valid_depth_only=True):
        n = w * h
        pts, nrm, col = (np.empty((n, 3), np.float32) for _ in range(3))
        hit = np.empty(n, np.uint8)
        lib().orc_tsdf_raycast(_p(self.tw), _p(self.col), C.c_float(self.length), C.c_int(self.res), C.c_int(self.ct),
                               _p(self.origin), C.c_int(w), C.c_int(h), _p(k4(K)), _p(_f(E, 16)), C.c_float(sdf_trunc), _p(pts),
                               _p(nrm), _p(col), _p(hit))
        if project_valid_depth_only:
            k = hit.astype(bool)
            return pts[k], nrm[k], col[k]
        return pts, nrm, col

    def colors_rgb(self):
        """the colour planes as [N, 3] (Gray32's one plane repeated; None for NoColor)"""
        if self.ct == NO_COLOR:
            return None
        return np.repeat(self.col.T, 3, 1) if self.ct == GRAY32 else self.col.T.copy()
