"""PointCloud::CreateFromDepthImage / CreateFromRGBDImage through the C++ facade (tests/cpp/facade_depth_cloud.cpp):
compiles and links with plain g++ (CPU); on the GPU its argument errors throw and a uint16 sphere view with random RGB
colour gives the oracle's rows bit for bit (strided depth, and RGB-D with a cutoff, normals and both
project_valid_depth_only values)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_depth_cloud_compiles_and_links():
    exe = build_facade("facade_depth_cloud")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_depth_cloud_matches_oracle():
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    from oracle import depth_cloud_py as D
    from oracle import tsdf_py as T
    exe = build_facade("facade_depth_cloud")
    w, h = 99, 73
    K, E = ring_cameras(4, w, h)[1]
    E = E.copy()
    E[:3, :3] *= np.float32(1.1)  # non-rigid
    depth = np.round(sphere_depth(K, ring_cameras(4, w, h)[1][1], w, h, 0.8) * 1000).astype(np.uint16)
    color = np.random.default_rng(2).integers(0, 256, (h, w, 3), dtype=np.uint8)
    with tempfile.TemporaryDirectory() as d:
        np.concatenate([[w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]], E.reshape(16)]).astype(np.float32).tofile(os.path.join(d, "params.f32"))
        depth.tofile(os.path.join(d, "depth.u16"))
        color.tofile(os.path.join(d, "color.u8"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        got = {n: np.fromfile(os.path.join(d, "out_%s.f32" % n), np.float32).reshape(-1, 3)
               for n in ("d_points", "v_points", "v_normals", "v_colors", "a_points", "a_colors")}

    def same(a, b):
        np.testing.assert_array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
    same(got["d_points"], D.depth_to_points(depth, K, E, 1000.0, 4.0, 3)[0])
    f = T.depth_to_float(depth, 1000.0, 4.0)
    p, n, c = D.depth_to_points(f, K, E, color=color, depth_cutoff=2.0, compute_normals=True)
    same(got["v_points"], p), same(got["v_normals"], n), same(got["v_colors"], c)
    p, _, c = D.depth_to_points(f, K, E, color=color, depth_cutoff=2.0, project_valid_depth_only=False)
    same(got["a_points"], p), same(got["a_colors"], c)
    assert len(got["v_points"]) > 500
