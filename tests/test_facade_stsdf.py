"""ScalableTSDFVolume through the C++ facade (tests/cpp/facade_stsdf.cpp): compiles and links with plain g++ (CPU); on
the GPU its argument errors throw and an RGB8 volume grown from map_size 1 over four sphere views gives the oracle's
ExtractPointCloud and ExtractVoxelPointCloud bit for bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_stsdf_compiles_and_links():
    exe = build_facade("facade_stsdf")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_stsdf_matches_oracle():
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    from oracle import stsdf_py as S
    from oracle import tsdf_py as T
    exe = build_facade("facade_stsdf")
    w, h, vl, trunc = 96, 72, 1.0 / 64, 0.04
    cams = ring_cameras(4, w, h)
    K = cams[0][0]
    depth = np.stack([np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16) for _, E in cams])
    color = np.random.default_rng(4).integers(0, 256, (len(cams), h, w, 3), dtype=np.uint8)
    ref = S.Volume(vl, trunc, S.RGB8, 4)
    for f, (_, E) in enumerate(cams):
        ref.integrate(T.depth_to_float(depth[f], 1000.0, 4.0), color[f], K, E)
    with tempfile.TemporaryDirectory() as d:
        np.concatenate([[w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], len(cams), vl, trunc]] +
                       [E.reshape(16) for _, E in cams]).astype(np.float32).tofile(os.path.join(d, "params.f32"))
        depth.tofile(os.path.join(d, "depth.u16"))
        color.tofile(os.path.join(d, "color.u8"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        got = {n: np.fromfile(os.path.join(d, "out_%s.f32" % n), np.float32).reshape(-1, 3)
               for n in ("points", "normals", "colors", "vpoints", "vcolors")}

    def same(a, b):
        np.testing.assert_array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
    p, n, c = ref.extract_point_cloud()
    same(got["points"], p), same(got["normals"], n), same(got["colors"], c)
    vp, vc = ref.extract_voxel_point_cloud()
    same(got["vpoints"], vp), same(got["vcolors"], vc)
    assert len(p) > 100
