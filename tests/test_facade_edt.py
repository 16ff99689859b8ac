"""geometry::DistanceTransform through the C++ facade (tests/cpp/facade_edt.cpp): compiles and links with plain g++ (CPU);
on the GPU illegal resolutions throw, a voxel-size mismatch is logged and changes nothing, and ComputeEDT, GetDistances
and GetVoxel equal the oracle."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT


def build_facade():
    import __graft_entry__
    __graft_entry__.build()
    from test_facade_cpp import build_dir
    exe = os.path.join(build_dir(), "facade_edt")
    lib = os.path.join(ROOT, "cupoch_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_edt.cpp"), "-o", exe, "-L" + lib,
                           "-lcupoch_b200", "-Wl,-rpath," + lib])
    return exe


def test_facade_edt_compiles_and_links():
    exe = build_facade()
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_edt_matches_oracle():
    from oracle import edt_py
    exe = build_facade()
    r, vs, origin = 40, 0.25, np.array([0.5, -1.0, 2.0], np.float32)
    rng = np.random.default_rng(5)
    cells = rng.integers(-3, r + 3, (300, 3)).astype(np.int32)  # some outside the grid
    q = (rng.uniform(-6, 6, (2000, 3)) + origin).astype(np.float32)
    q[:3] = [[np.nan, 0, 0], [100, 0, 0], origin]
    with tempfile.TemporaryDirectory() as d:
        np.array([vs, r, *origin], np.float32).tofile(os.path.join(d, "params.f32"))
        cells.tofile(os.path.join(d, "cells.i32"))
        q.tofile(os.path.join(d, "queries.f32"))
        res = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        assert "Unsupport computing Voronoi diagrams from different voxel size." in res.stderr
        dist = np.fromfile(os.path.join(d, "out_dist.f32"), np.float32)
        vox = np.fromfile(os.path.join(d, "out_voxel.i32"), np.int32).reshape(-1, 6)
    nearest, state, o_dist = edt_py.compute(r, cells, vs)
    np.testing.assert_array_equal(dist.view(np.uint32), edt_py.get_distances(o_dist, q, vs, origin, ).view(np.uint32))
    idx = edt_py.voxel_index(q, vs, origin, r)
    found = idx >= 0
    np.testing.assert_array_equal(vox[:, 0], found.astype(np.int32))
    i = np.maximum(idx, 0)
    np.testing.assert_array_equal(vox[found, 1:4], nearest.reshape(-1, 3)[i[found]].astype(np.int32))
    np.testing.assert_array_equal(vox[found, 4], state.reshape(-1)[i[found]].astype(np.int32))
    np.testing.assert_array_equal(vox[found, 5], o_dist.reshape(-1)[i[found]].view(np.int32))
    np.testing.assert_array_equal(vox[~found], np.tile([0, 0, 0, 0, 2, 0], ((~found).sum(), 1)))
    assert found.sum() > 1000 and (~found).sum() >= 2
