"""collision::ComputeIntersection through the C++ facade (tests/cpp/facade_collision.cpp): compiles and links with plain
g++ (CPU); on the GPU the reference's VoxelVoxel test passes with its keys assigned to voxels_keys_, and the pairs of
VoxelGrid x VoxelGrid, VoxelGrid x primitives (both orders) and OccupancyGrid x VoxelGrid (both orders) equal the
oracle's."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade
from test_oracle_collision import random_prims


def test_facade_collision_compiles_and_links():
    exe = build_facade("facade_collision")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_collision_matches_oracle():
    from oracle import collision_py as OC
    exe = build_facade("facade_collision")
    rng = np.random.default_rng(9)
    ka = np.floor(rng.normal(20, 6, (3000, 3))).astype(np.int32)
    kb = np.floor(rng.normal(15, 5, (2000, 3))).astype(np.int32)
    va, oa, vb, ob, margin = 0.05, [0.01, -0.02, 0.03], 0.07, [-0.04, 0.02, 0.0], 0.03
    recs = random_prims(rng, 200, 1.5, 0.05)
    occ_vs, occ_res = 0.05, 64
    cells = np.unique(rng.integers(32, 64, (2000, 3)), axis=0).astype(np.int32)
    with tempfile.TemporaryDirectory() as d:
        np.array([va, *oa, vb, *ob, margin, occ_vs, occ_res], np.float32).tofile(os.path.join(d, "params.f32"))
        ka.tofile(os.path.join(d, "keys_a.i32"))
        kb.tofile(os.path.join(d, "keys_b.i32"))
        cells.tofile(os.path.join(d, "occ_cells.i32"))
        np.concatenate([np.concatenate([[r["type"]], r["transform"], r["lengths"], [r["radius"], r["height"]]]) for r in recs]
                       ).astype(np.float32).tofile(os.path.join(d, "prims.f32"))
        res = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        out = {k: np.fromfile(os.path.join(d, "out_%s.i32" % k), np.int32).reshape(-1, 2) for k in ("ab", "ap", "pa", "ob", "bo")}
    A, B, P = OC.voxel_grid(ka, va, oa), OC.voxel_grid(kb, vb, ob), OC.prims(recs)
    prob = np.full((occ_res,) * 3, np.nan, np.float32)
    prob[tuple(cells.T)] = 0.85
    lo, hi = np.minimum(cells.min(0), occ_res // 2), np.maximum(cells.max(0), occ_res // 2)  # the box starts at the centre cell
    O = OC.occupancy_grid(prob, lo, hi, 0.0, occ_vs, [0, 0, 0])
    want = {"ab": OC.compute(A, B, margin), "ap": OC.compute(A, P, margin), "pa": OC.compute(P, A, margin),
            "ob": OC.compute(O, B, margin), "bo": OC.compute(B, O, margin)}
    for k in want:
        np.testing.assert_array_equal(out[k], want[k], err_msg=k)
    assert all(len(v) for v in want.values())
