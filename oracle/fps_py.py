"""ctypes loader for the FarthestPointDownSample restatement (oracle/fps.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --fps, never by the product package
cupoch_b200/.  The library is compiled on first use with oracle/Makefile's flags into oracle/_build/ (or a per-user
temporary directory when the tree is read-only).
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "fps.c")
CFLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wextra"]


def build(force=False):
    out_dir = os.path.join(_HERE, "_build")
    if not os.access(_HERE, os.W_OK) and not os.access(out_dir, os.W_OK):
        out_dir = os.path.join(tempfile.gettempdir(), "cphb_oracle_%d" % os.getuid())
    so = os.path.join(out_dir, "libfps.so")
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


def farthest_point_down_sample(pts, num_samples):
    """-> (indices [num_samples] int32, final running distances [n] float32); the loop runs for any num_samples
    (DESIGN.md arithmetic contract, smallest index among equal distances).  No points: nothing to pick, both empty."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    n, k = len(pts), int(num_samples)
    if n == 0:
        return np.empty(0, np.int32), np.empty(0, np.float32)
    idx = np.empty(k, np.int32)
    dist = np.empty(n, np.float32)
    lib().orc_farthest_point_down_sample(_p(pts), C.c_int(n), C.c_long(k), _p(idx), _p(dist))
    return idx, dist
