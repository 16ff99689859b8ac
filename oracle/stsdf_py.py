"""ctypes loader for the ScalableTSDFVolume restatement (oracle/stsdf.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/, never by the product package cupoch_b200/.  The
library is built by oracle.build("stsdf") (oracle/__init__.py's recipe).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

NO_COLOR, RGB8, GRAY32 = 0, 1, 2
PLANES = {NO_COLOR: 0, RGB8: 3, GRAY32: 1}
_lib = None


def build(force=False):
    return _build("stsdf", force)


def lib():
    global _lib
    if _lib is None:
        _lib = load("stsdf")
        _lib.orc_st_create.restype = C.c_void_p
        _lib.orc_st_create.argtypes = [C.c_float, C.c_float, C.c_int, C.c_int]
        for f in ("orc_st_destroy", "orc_st_reset", "orc_st_data"):
            getattr(_lib, f).restype = None
        for f in ("orc_st_units", "orc_st_extract_points", "orc_st_extract_voxels"):
            getattr(_lib, f).restype = C.c_longlong
        _lib.orc_st_integrate.restype = C.c_int
    return _lib


def unpack(keys):
    """packed keys -> [n, 3] int64 unit keys"""
    k = np.asarray(keys, np.uint64)
    return np.stack([((k >> np.uint64(42 - 21 * a)) & np.uint64(0x1fffff)).astype(np.int64) - (1 << 20) for a in range(3)], 1)


class Volume:
    def __init__(self, voxel_length, sdf_trunc, color_type=NO_COLOR, depth_sampling_stride=4):
        self.ct = int(color_type)
        self.vl = np.float32(voxel_length)
        self._h = C.c_void_p(lib().orc_st_create(C.c_float(voxel_length), C.c_float(sdf_trunc), C.c_int(self.ct),
                                                 C.c_int(depth_sampling_stride)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_st_destroy(self._h)
            self._h = None

    def reset(self):
        lib().orc_st_reset(self._h)

    def integrate(self, depth, color, K, E):
        """depth: float32 [h, w] metres; color: uint8 [h, w, 3] (RGB8), float32 [h, w] (Gray32) or None"""
        d = np.ascontiguousarray(depth, np.float32)
        h, w = d.shape
        c = None if color is None or self.ct == NO_COLOR else np.ascontiguousarray(color)
        K = np.asarray(K, np.float32).reshape(3, 3)
        K4 = np.float32([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
        E = np.ascontiguousarray(np.asarray(E, np.float32).reshape(16))
        rc = lib().orc_st_integrate(self._h, _p(d), _p(c), C.c_int(w), C.c_int(h), _p(K4), _p(E))
        if rc == -1:
            raise ValueError("the extrinsic is not invertible")
        if rc == -2:
            raise ValueError("a unit key is out of range")

    def units(self):
        """(keys [u] uint64, tw [u, 4096, 2], col [u, planes, 4096])"""
        u = lib().orc_st_units(self._h)
        keys, tw = np.empty(u, np.uint64), np.empty((u, 4096, 2), np.float32)
        col = np.empty((u, PLANES[self.ct], 4096), np.float32)
        lib().orc_st_data(self._h, _p(keys), _p(tw), _p(col))
        return keys, tw, col

    def extract_point_cloud(self):
        L = lib()
        m = L.orc_st_extract_points(self._h, None, None, None)
        pts, nrm, col = (np.empty((max(m, 1), 3), np.float32) for _ in range(3))
        L.orc_st_extract_points(self._h, _p(pts), _p(nrm), _p(col))
        return pts[:m], nrm[:m], (col[:m] if self.ct != NO_COLOR else None)

    def extract_voxel_point_cloud(self):
        L = lib()
        m = L.orc_st_extract_voxels(self._h, None, None)
        pts, col = np.empty((max(m, 1), 3), np.float32), np.empty((max(m, 1), 3), np.float32)
        L.orc_st_extract_voxels(self._h, _p(pts), _p(col))
        return pts[:m], col[:m]
