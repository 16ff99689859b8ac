"""UniformTSDFVolume and RGBDImage through the C++ facade (tests/cpp/facade_tsdf.cpp): compiles and links with plain g++
(CPU); on the GPU its known answers hold and an RGB8 volume integrated from four sphere views gives the oracle's
ExtractPointCloud, ExtractVoxelPointCloud, ExtractVoxelGrid and Raycast (both project_valid_depth_only values), bit for
bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_tsdf_compiles_and_links():
    exe = build_facade("facade_tsdf")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_tsdf_matches_oracle():
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    from oracle import tsdf_py as T
    exe = build_facade("facade_tsdf")
    w, h, length, res, trunc = 96, 72, 2.0, 96, 0.06
    cams = ring_cameras(4, w, h)
    K = cams[0][0]
    rng = np.random.default_rng(4)
    depth = np.stack([np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16) for _, E in cams])
    color = rng.integers(0, 256, (len(cams), h, w, 3), dtype=np.uint8)
    ref = T.Volume(length, res, trunc, T.RGB8)
    for f, (_, E) in enumerate(cams):
        ref.integrate(T.depth_to_float(depth[f], 1000.0, 100.0), color[f], K, E)
    with tempfile.TemporaryDirectory() as d:
        np.concatenate([[w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], len(cams), length, res, trunc]] +
                       [E.reshape(16) for _, E in cams]).astype(np.float32).tofile(os.path.join(d, "params.f32"))
        depth.tofile(os.path.join(d, "depth.u16"))
        color.tofile(os.path.join(d, "color.u8"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr

        def rd(name, dt=np.float32):
            return np.fromfile(os.path.join(d, "out_%s" % name), dt).reshape(-1, 3)
        got = {n: rd(n + ".f32") for n in ("points", "normals", "colors", "vpoints", "vcolors", "vg_colors")}
        keys = rd("vg_keys.i32", np.int32)
        org = np.fromfile(os.path.join(d, "out_vg_origin.f32"), np.float32)
        rays = {(v, n): rd("ray_%s_%s.f32" % (v, n)) for v in ("valid", "all") for n in ("points", "normals", "colors")}

    def same(a, b):
        np.testing.assert_array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
    p, n, c = ref.extract_point_cloud()
    same(got["points"], p), same(got["normals"], n), same(got["colors"], c)
    vp, vc = ref.extract_voxel_point_cloud()
    same(got["vpoints"], vp), same(got["vcolors"], vc)
    rk, rc, vs, ro = ref.extract_voxel_grid()
    np.testing.assert_array_equal(keys, rk)
    same(got["vg_colors"], rc), same(org, np.append(ro, vs))
    for v, valid in (("valid", True), ("all", False)):
        rp, rn, rcol = ref.raycast(K, cams[0][1], w, h, trunc, valid)
        same(rays[v, "points"], rp), same(rays[v, "normals"], rn), same(rays[v, "colors"], rcol)
    assert len(p) > 100 and len(rays["valid", "points"]) > 100
