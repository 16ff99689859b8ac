"""PointCloud::SegmentPlane through the C++ facade (tests/cpp/facade_segment_plane.cpp): compiles and links with plain
g++ (CPU); on the GPU it passes the reference's known-answer test and, after srand(), equals the oracle given the
same rand() draws."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from cupoch_b200.testing import datagen
from test_facade_cpp import build_facade


@pytest.fixture(scope="module")
def seg():
    """the SegmentPlane restatement (oracle/segment_plane.c)"""
    from oracle import segment_plane_py
    segment_plane_py.build()
    return segment_plane_py


def test_facade_segment_plane_compiles_and_links():
    exe = build_facade("facade_segment_plane")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_segment_plane_matches_oracle(seg):
    exe = build_facade("facade_segment_plane")
    pts =datagen.plane_scene(50_000, 17)
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
