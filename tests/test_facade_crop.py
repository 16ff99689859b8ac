"""Bounding boxes and point-cloud cleanup through the C++ facade (tests/cpp/facade_crop.cpp): compiles and links with
plain g++ (CPU); on the GPU the reference's known box and the argument rules hold, and every call's output equals the
oracle's (oracle/crop.c)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from cupoch_b200.testing import datagen
from test_facade_cpp import build_facade


@pytest.fixture(scope="module")
def cp():
    from oracle import crop_py
    crop_py.build()
    return crop_py


def test_facade_crop_compiles_and_links():
    exe = build_facade("facade_crop")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_crop_matches_oracle(cp):
    exe = build_facade("facade_crop")
    n = 200_000
    pts = datagen.uniform_cube(n, 61, hi=(4, 4, 1))
    pts[::101, 1] = np.nan
    pts[50::211, 2] = np.inf
    nrm = datagen.unit_normals(n, 62) * np.float32(3)
    nrm[::97] = 0
    with tempfile.TemporaryDirectory() as d:
        pts.tofile(os.path.join(d, "points.f32"))
        nrm.tofile(os.path.join(d, "normals.f32"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr

        def rd(name):
            return np.fromfile(os.path.join(d, name + ".f32"), np.float32)
        got = {k: rd(k) for k in ("crop_aabb", "crop_obb", "pass_through", "uniform", "finite", "obb", "normalized", "oriented")}
    R = np.float32([[0.8660254, -0.5, 0], [0.5, 0.8660254, 0], [0, 0, 1]])
    box = cp.obb_box_points((2, 2, 0.5), R, (2.6, 2.6, 1.2))
    np.testing.assert_array_equal(got["crop_aabb"].reshape(-1, 3), pts[cp.aabb_indices(pts, (0.5, 1, 0.25), (2, 4, 0.75))])
    np.testing.assert_array_equal(got["crop_obb"].reshape(-1, 3), pts[cp.obb_indices(pts, box)])
    np.testing.assert_array_equal(got["pass_through"].reshape(-1, 3), pts[cp.pass_through_indices(pts, 1, 0.25, 0.75)])
    np.testing.assert_array_equal(got["uniform"].reshape(-1, 3), pts[cp.uniform_rows(n, 5)])
    np.testing.assert_array_equal(got["finite"].reshape(-1, 3), pts[cp.finite_indices(pts)])
    c, Rb, e = cp.obb_create(pts)
    np.testing.assert_array_equal(got["obb"], np.concatenate([c, Rb.reshape(-1), e]))
    np.testing.assert_array_equal(got["normalized"].reshape(-1, 3), cp.normalize_normals(nrm))
    np.testing.assert_array_equal(got["oriented"].reshape(-1, 3), cp.orient_normals(nrm, (0, 0.5, 2)))
