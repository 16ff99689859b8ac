"""The VoxelGrid operations through the C++ facade (tests/cpp/facade_voxelgrid_ops.cpp): compiles and links with plain
g++ (CPU); on the GPU its known answers hold and CheckIfIncluded, +=, AddVoxels, SelectByIndex (both), PaintIndexedColor,
CarveDepthMap of a dense 64^3 grid and both CreateFromOccupancyGrid calls equal the oracle's, bit for bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_voxelgrid_ops_compiles_and_links():
    exe = build_facade("facade_voxelgrid_ops")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_voxelgrid_ops_match_oracle():
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    from oracle import voxelgrid_ops_py as V
    exe = build_facade("facade_voxelgrid_ops")
    rng = np.random.default_rng(12)
    vs, o = 0.05, np.float32([0.01, -0.02, 0.03])
    ka = np.unique(rng.integers(0, 30, (20000, 3)), axis=0).astype(np.int32)
    kb = np.unique(rng.integers(15, 45, (20000, 3)), axis=0).astype(np.int32)
    ca, cb = rng.random((len(ka), 3)).astype(np.float32), rng.random((len(kb), 3)).astype(np.float32)
    q = (rng.uniform(-0.2, 1.7, (50000, 3)) + o).astype(np.float32)
    q[:10, 0] = np.nan
    idx = rng.integers(0, len(ka), 3000).astype(np.int64)
    w, h = 96, 72
    K, E = ring_cameras(3, w, h)[1]
    depth = sphere_depth(K, E, w, h, 0.8)
    occ_vs, occ_res = 0.05, 64
    cells = np.unique(rng.integers(20, 50, (3000, 3)), axis=0).astype(np.int32)
    with tempfile.TemporaryDirectory() as d:
        np.concatenate([[vs, *o, occ_vs, occ_res, w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]], E.reshape(16)]).astype(np.float32).tofile(
            os.path.join(d, "params.f32"))
        for name, a in (("keys_a.i32", ka), ("keys_b.i32", kb), ("colors_a.f32", ca), ("colors_b.f32", cb), ("queries.f32", q),
                        ("idx.i64", idx), ("depth.f32", depth), ("occ_cells.i32", cells)):
            a.tofile(os.path.join(d, name))
        res = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr

        def grid(name):
            return (np.fromfile(os.path.join(d, "out_%s_keys.i32" % name), np.int32).reshape(-1, 3),
                    np.fromfile(os.path.join(d, "out_%s_colors.f32" % name), np.float32).reshape(-1, 3))
        out = {n: grid(n) for n in ("merge", "add", "select", "invert", "paint", "carve", "occvg")}
        included = np.fromfile(os.path.join(d, "out_included.u8"), np.uint8).astype(bool)
        occ_origin = np.fromfile(os.path.join(d, "out_occvg_origin.f32"), np.float32)
        pts = np.fromfile(os.path.join(d, "out_occpc_points.f32"), np.float32).reshape(-1, 3)
        pcols = np.fromfile(os.path.join(d, "out_occpc_colors.f32"), np.float32).reshape(-1, 3)
    dense = V.create_dense(2.0 / 64, 2, 2, 2)
    o_dense = np.float32([-1, -1, -1])
    blue = np.tile(np.float32([0, 0, 1]), (len(cells), 1))
    want = {"merge": V.merge(ka, ca, kb, cb, True), "add": V.merge(ka, ca, kb, cb, False), "select": V.select(ka, ca, idx),
            "invert": V.select(ka, ca, idx, True), "paint": (ka, V.paint(ca, idx, (0.25, 0.5, 0.75))),
            "carve": V.carve(*dense, 2.0 / 64, o_dense, depth, K, E, False), "occvg": (cells, blue)}
    for n, (wk, wc) in want.items():
        np.testing.assert_array_equal(out[n][0], wk, err_msg=n)
        np.testing.assert_array_equal(out[n][1].view(np.uint32), np.asarray(wc, np.float32).view(np.uint32), err_msg=n)
    assert 0 < len(want["carve"][0]) < 64 ** 3
    np.testing.assert_array_equal(included, V.check_if_included(ka, vs, o, q))
    np.testing.assert_array_equal(occ_origin, V.occ_voxel_origin(occ_res, occ_vs, [0, 0, 0]))
    np.testing.assert_array_equal(pts.view(np.uint32), V.occ_points(cells, occ_res, occ_vs, [0, 0, 0]).view(np.uint32))
    np.testing.assert_array_equal(pcols, blue)
