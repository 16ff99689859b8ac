"""ctypes loader for the SegmentPlane restatement (oracle/segment_plane.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --segment-plane, never by the
product package cupoch_b200/.  The library is compiled on first use with oracle/Makefile's flags into oracle/_build/
(or a per-user temporary directory when the tree is read-only).
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "segment_plane.c")
CFLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wextra"]


def build(force=False):
    out_dir = os.path.join(_HERE, "_build")
    if not os.access(_HERE, os.W_OK) and not os.access(out_dir, os.W_OK):
        out_dir = os.path.join(tempfile.gettempdir(), "cphb_oracle_%d" % os.getuid())
    so = os.path.join(out_dir, "libsegment_plane.so")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(_SRC):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-shared", "-o", so, _SRC, "-lm"])
    return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def segment_plane(pts, distance_threshold, ransac_n, seeds):
    """PointCloud::SegmentPlane (segmentation.cu:187-267) with one seed per iteration ->
    (plane float32[4], ascending inlier indices int32, best iteration or -1, fitness, inlier_rmse)"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    seeds = np.ascontiguousarray(seeds, np.int32).reshape(-1)
    plane, fr = np.zeros(4, np.float32), np.zeros(2, np.float32)
    idx = np.empty(max(len(pts), 1), np.int32)
    m, best = C.c_int(0), C.c_int(-1)
    rc = lib().orc_segment_plane(_p(pts), C.c_int(len(pts)), C.c_float(distance_threshold), C.c_int(ransac_n),
                                 C.c_int(len(seeds)), _p(seeds), _p(plane), _p(idx), C.byref(m), C.byref(best), _p(fr))
    assert rc == 0
    return plane, idx[:m.value].copy(), int(best.value), np.float32(fr[0]), np.float32(fr[1])


def ransac_keys(seed, n):
    keys = np.empty(n, np.int32)
    lib().orc_ransac_keys(C.c_int32(seed), C.c_int(n), _p(keys))
    return keys


def ransac_samples(n, seeds):
    """-> [T, 3] int32: d_cards[0..2] after each iteration's stable sort"""
    seeds = np.ascontiguousarray(seeds, np.int32).reshape(-1)
    out = np.empty((len(seeds), 3), np.int32)
    lib().orc_ransac_samples(C.c_int(n), C.c_int(len(seeds)), _p(seeds), _p(out))
    return out
