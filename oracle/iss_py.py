"""ctypes loader for the ComputeISSKeypoints restatement (oracle/iss.c, compiled together with oracle/oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/bench_ops.py --iss, never by the product package
cupoch_b200/.  The library is compiled on first use with oracle/Makefile's flags into oracle/_build/ (or a per-user
temporary directory when the tree is read-only).
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "iss.c")
_DEPS = [_SRC, os.path.join(_HERE, "oracle.c"), os.path.join(_HERE, "oracle.h")]
CFLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wextra", "-Wno-unused-parameter",
          "-Wno-unused-function", "-Wno-unknown-pragmas"]


def build(force=False):
    out_dir = os.path.join(_HERE, "_build")
    if not os.access(_HERE, os.W_OK) and not os.access(out_dir, os.W_OK):
        out_dir = os.path.join(tempfile.gettempdir(), "cphb_oracle_%d" % os.getuid())
    so = os.path.join(out_dir, "libiss.so")
    if force or not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(p) for p in _DEPS):
        os.makedirs(out_dir, exist_ok=True)
        cmd = [os.environ.get("CC", "gcc")] + CFLAGS + ["-shared", "-o", so, _SRC, "-lm"]
        # OpenMP only parallelises over points (each point's result is computed alone): single-threaded if unavailable
        if subprocess.run(cmd[:1] + ["-fopenmp"] + cmd[1:], capture_output=True).returncode != 0:
            subprocess.check_call(cmd)
    return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_iss_keypoints.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def iss_keypoints(pts, salient_radius=0.0, non_max_radius=0.0, gamma_21=0.975, gamma_32=0.975, min_neighbors=5,
                  max_neighbors=100):
    """-> (mask [n] bool, saliency [n] float32, radii used float32[2]); both radii are replaced by 6 and 4 times the
    resolution when either is 0."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    n = len(pts)
    mask = np.zeros(max(n, 1), np.uint8)
    sal = np.zeros(max(n, 1), np.float32)
    radii = np.zeros(2, np.float32)
    rc = lib().orc_iss_keypoints(_p(pts), C.c_int(n), C.c_float(salient_radius), C.c_float(non_max_radius),
                                 C.c_float(gamma_21), C.c_float(gamma_32), C.c_int(min_neighbors), C.c_int(max_neighbors),
                                 _p(mask), _p(sal), _p(radii))
    if rc < 0:
        raise ValueError("max_neighbors must lie in [0, 256]")
    return mask[:n].astype(bool), sal[:n], radii
