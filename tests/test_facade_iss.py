"""geometry::keypoint::ComputeISSKeypoints through the C++ facade (tests/cpp/facade_iss.cpp): compiles and links with plain
g++ (CPU); on the GPU its empty and illegal-argument results hold and its keypoints, normals and mask equal the oracle's."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from cupoch_b200.testing import datagen


def build_facade():
    import __graft_entry__
    __graft_entry__.build()
    from test_facade_cpp import build_dir
    exe = os.path.join(build_dir(), "facade_iss")
    lib = os.path.join(ROOT, "cupoch_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_iss.cpp"), "-o", exe, "-L" + lib,
                           "-lcupoch_b200", "-Wl,-rpath," + lib])
    return exe


def test_facade_iss_compiles_and_links():
    exe = build_facade()
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_iss_matches_oracle():
    from oracle import iss_py
    exe = build_facade()
    pts, nrm = datagen.surface(60_000, 23)
    with tempfile.TemporaryDirectory() as d:
        pts.tofile(os.path.join(d, "points.f32"))
        nrm.tofile(os.path.join(d, "normals.f32"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "Input PointCloud is empty" in r.stderr and "max_neighbors must lie in [0, 256]" in r.stderr
        out_p = np.fromfile(os.path.join(d, "out_points.f32"), np.float32).reshape(-1, 3)
        out_n = np.fromfile(os.path.join(d, "out_normals.f32"), np.float32).reshape(-1, 3)
        mask = np.fromfile(os.path.join(d, "out_mask.u8"), np.uint8).astype(bool)
    o_mask, _, _ = iss_py.iss_keypoints(pts)
    assert o_mask.sum() > 0
    np.testing.assert_array_equal(mask, o_mask)
    np.testing.assert_array_equal(out_p, pts[o_mask])
    np.testing.assert_array_equal(out_n, nrm[o_mask])
