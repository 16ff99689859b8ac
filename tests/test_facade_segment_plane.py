"""PointCloud::SegmentPlane through the C++ facade (tests/cpp/facade_segment_plane.cpp): compiles and links with plain
g++ (CPU); on the GPU it passes the reference's known-answer test and, after srand(), equals the oracle given the
same rand() draws."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from cupoch_b200.testing import datagen


@pytest.fixture(scope="module")
def seg():
    """the SegmentPlane restatement (oracle/segment_plane.c)"""
    from oracle import segment_plane_py
    segment_plane_py.build()
    return segment_plane_py


def build_facade():
    import __graft_entry__
    __graft_entry__.build()
    exe = os.path.join(ROOT, "tests", "cpp", "_build", "facade_segment_plane")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    lib = os.path.join(ROOT, "cupoch_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_segment_plane.cpp"), "-o", exe, "-L" + lib,
                           "-lcupoch_b200", "-Wl,-rpath," + lib])
    return exe


def test_facade_segment_plane_compiles_and_links():
    exe = build_facade()
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_segment_plane_matches_oracle(seg):
    exe = build_facade()
    pts = datagen.plane_scene(50_000, 17)
    seed, thr, T = 3, 0.01, 50
    libc = C.CDLL(None)
    libc.srand(C.c_uint(seed))
    seeds = np.array([libc.rand() for _ in range(T)], np.int32)
    with tempfile.TemporaryDirectory() as d:
        pts.tofile(os.path.join(d, "points.f32"))
        r = subprocess.run([exe, d, str(seed), str(thr), str(T)], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        plane = np.fromfile(os.path.join(d, "plane.f32"), np.float32)
        idx = np.fromfile(os.path.join(d, "inliers.i64"), np.int64)
    o_plane, o_idx, _, _, _ = seg.segment_plane(pts, thr, 3, seeds)
    np.testing.assert_array_equal(plane, o_plane)
    np.testing.assert_array_equal(idx, o_idx)
