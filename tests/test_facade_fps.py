"""PointCloud::FarthestPointDownSample through the C++ facade (tests/cpp/facade_fps.cpp): compiles and links with plain
g++ (CPU); on the GPU its shortcuts hold and its picks and gathered normals equal the oracle's."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from cupoch_b200.testing import datagen
from test_facade_cpp import build_facade


@pytest.fixture(scope="module")
def fpso():
    """the FarthestPointDownSample restatement (oracle/fps.c)"""
    from oracle import fps_py
    fps_py.build()
    return fps_py


def test_facade_fps_compiles_and_links():
    exe = build_facade("facade_fps")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_fps_matches_oracle(fpso):
    exe = build_facade("facade_fps")
    pts, nrm = datagen.surface(60_000, 19)
    k = 700
    with tempfile.TemporaryDirectory() as d:
        pts.tofile(os.path.join(d, "points.f32"))
        nrm.tofile(os.path.join(d, "normals.f32"))
        r = subprocess.run([exe, d, str(k)], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "Illegal number of samples" in r.stderr
        out_p = np.fromfile(os.path.join(d, "out_points.f32"), np.float32).reshape(-1, 3)
        out_n = np.fromfile(os.path.join(d, "out_normals.f32"), np.float32).reshape(-1, 3)
    o_idx, _ = fpso.farthest_point_down_sample(pts, k)
    np.testing.assert_array_equal(out_p, pts[o_idx])
    np.testing.assert_array_equal(out_n, nrm[o_idx])
