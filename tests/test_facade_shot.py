"""registration::ComputeSHOTFeature through the C++ facade (tests/cpp/facade_shot.cpp): compiles and links with plain g++
(CPU); on the GPU its empty and illegal-argument results hold and its descriptors equal the oracle's bit for bit."""
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
    exe = os.path.join(build_dir(), "facade_shot")
    lib = os.path.join(ROOT, "cupoch_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_shot.cpp"), "-o", exe, "-L" + lib,
                           "-lcupoch_b200", "-Wl,-rpath," + lib])
    return exe


def test_facade_shot_compiles_and_links():
    exe = build_facade()
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_shot_matches_oracle():
    from oracle import shot_py
    exe = build_facade()
    pts, nrm = datagen.surface(20_000, 29)
    radius = np.float32(5.0 / np.sqrt(1e5))
    with tempfile.TemporaryDirectory() as d:
        pts.tofile(os.path.join(d, "points.f32"))
        nrm.tofile(os.path.join(d, "normals.f32"))
        np.array([radius], np.float32).tofile(os.path.join(d, "radius.f32"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "input point cloud has no normal" in r.stderr and "knn must be <= 100" in r.stderr
        got = np.fromfile(os.path.join(d, "out_shot.f32"), np.float32).reshape(-1, 352)
    want = shot_py.compute_shot_feature(pts, nrm, float(radius), 0, float(radius), 100)
    assert (np.abs(want).sum(1) > 0).mean() > 0.9
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
