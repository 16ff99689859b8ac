"""GPU: collision::ComputeIntersection (csrc/collision.cu) through cph.collision.compute_intersection.

- The device's pairs are identical to the brute-force oracle's (oracle/collision.c) for all seven operand pairs, at
  0, 1, 1 k and 100 k elements, margins 0, 0.5 and 3 voxels, different voxel sizes and origins that do not line up,
  duplicate and unsorted keys, exact tie geometry, OccupancyGrids after insert and after set_free_area, one primitive
  whose region covers > 1e5 cells and 1e4 primitives.  A 2 M-voxel grid is checked on sampled queries.
- The reference's VoxelVoxel known answer; a fixed launch count; repeated calls are bit-identical; illegal arguments
  are refused."""
import ctypes as C
import json
import zlib

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from oracle import collision_py as OC
from test_oracle_collision import GOLD, big_rotated_box_scene, random_prims

G, K = cph.geometry, cph.collision


def vg(keys, vs, origin):
    g = G.VoxelGrid()
    g.voxel_size = float(vs)
    g.origin = np.asarray(origin, np.float32)
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, 3)
    g.voxels_keys = keys if len(keys) else None
    return g, OC.voxel_grid(keys, vs, origin)


def occ_cells(cells, vs, res, origin, free_area=None):
    o = G.OccupancyGrid(vs, res, origin)
    cells = np.ascontiguousarray(cells, np.int32).reshape(-1, 3)
    if len(cells):
        o.add_voxels(cells, True)
    if free_area is not None:
        o.set_free_area(*free_area)
    return o, occ_operand(o)


def occ_operand(o):
    prob = o.to_torch().cpu().numpy()
    lo, hi = o._bounds()
    return OC.occupancy_grid(prob, lo, hi, o.occ_prob_thres_log, o.voxel_size, o.origin)


def product_prim(rec):
    t, T = int(rec["type"]), np.asarray(rec["transform"], np.float32).reshape(4, 4)
    if t == OC.BOX:
        return K.Box(rec["lengths"], T)
    if t == OC.SPHERE:
        s = K.Sphere(float(rec["radius"]))
        s.transform = T
        return s
    if t == OC.CAPSULE:
        return K.Capsule(float(rec["radius"]), float(rec["height"]), T)
    return K.Cylinder(float(rec["radius"]), float(rec["height"]), T)


def prims(recs):
    return K.PrimitiveArray([product_prim(r) for r in recs]), OC.prims(recs) if len(recs) else np.zeros(0, OC.PRIM_DTYPE)


def check(a, b, margin):
    (pa, oa), (pb, ob) = a, b
    res = K.compute_intersection(pa, pb, margin)
    got = res.get_collision_index_pairs()
    want = OC.compute(oa, ob, margin)
    assert got.dtype == np.int32 and got.shape == want.shape and np.array_equal(got, want), (got[:5], want[:5])
    return got


def cluster_keys(rng, n, span):
    """n keys (unsorted, some repeated) of a few blobs inside [0, span)^3"""
    if n == 0:
        return np.zeros((0, 3), np.int32)
    c = rng.uniform(0, span, (4, 3))
    pts = c[rng.integers(0, 4, n)] + rng.normal(0, span / 8, (n, 3))
    return np.clip(np.floor(pts), -span, 2 * span).astype(np.int32)


VS_T, O_T = 0.05, (0.013, -0.021, 0.007)
VS_Q, O_Q = 0.07, (-0.031, 0.017, 0.044)
PAIRS = ["vg_vg", "vg_occ", "occ_vg", "vg_prim", "prim_vg", "occ_prim", "prim_occ"]


def make(kind, n, rng, vs, origin, span=None):
    if kind == "vg":
        span = span or max(4, int(round(n ** (1 / 3) * 2)))
        return vg(cluster_keys(rng, n, span), vs, origin)
    if kind == "occ":
        res = 64 if n <= 1000 else 128
        cells = np.unique(np.clip(cluster_keys(rng, n, res // 2) + res // 4, 0, res - 1), axis=0)
        return occ_cells(cells, vs, res, origin)
    return prims(random_prims(rng, n, 1.5, vs))


@pytest.mark.parametrize("margin_vs", [0.0, 0.5, 3.0])
@pytest.mark.parametrize("sizes", [(0, 7), (7, 0), (1, 1), (1000, 1000), (100_000, 1000), (1000, 100_000)])
@pytest.mark.parametrize("pair", PAIRS)
def test_pairs_match_oracle(pair, sizes, margin_vs):
    ka, kb = pair.split("_")
    na, nb = sizes
    if (ka == "prim" and na > 10_000) or (kb == "prim" and nb > 10_000):
        pytest.skip("1e4 primitives are in test_many_primitives")
    rng = np.random.default_rng(zlib.crc32(repr((pair, sizes, margin_vs)).encode()))
    a = make(ka, na, rng, VS_T, O_T)
    b = make(kb, nb, rng, VS_Q if ka != "prim" else VS_T, O_Q)
    check(a, b, margin_vs * VS_T)


def test_known_answer_voxel_voxel():
    g = json.load(open(GOLD))
    for step in g["steps"]:
        a, _ = vg(np.asarray(step["keys1"], np.int32).reshape(-1, 3), g["voxel_size"], g["origin"])
        b, _ = vg(np.asarray(step["keys2"], np.int32).reshape(-1, 3), g["voxel_size"], g["origin"])
        r = K.compute_intersection(a, b)
        assert r.is_collided() == step["collided"]
        assert (r.first, r.second) == (K.CollisionType.VoxelGrid, K.CollisionType.VoxelGrid)
        if "pairs" in step:
            assert r.get_collision_index_pairs().tolist() == step["pairs"]
            assert r.get_first_collision_indices().tolist() == [0] and r.get_second_collision_indices().tolist() == [0]


def test_duplicate_and_unsorted_keys():
    rng = np.random.default_rng(7)
    keys = cluster_keys(rng, 5000, 12)
    keys = np.concatenate([keys, keys[::-3], keys[:100]])
    rng.shuffle(keys)
    for m in (0.0, 0.5 * VS_T):
        check(vg(keys, VS_T, O_T), vg(cluster_keys(rng, 3000, 12), VS_T, O_T), m)
        check(vg(keys, VS_T, O_T), prims(random_prims(rng, 50, 12 * VS_T, VS_T)), m)


def test_tie_geometry():
    """voxel sizes that are powers of two and integer origins: touching faces, edges and tangent primitives"""
    k = np.stack(np.meshgrid(*[np.arange(0, 8, 2)] * 3, indexing="ij"), -1).reshape(-1, 3)
    for vs_q, o_q in ((0.5, (0.0, 0.0, 0.0)), (0.25, (1.0, 0.0, -1.0)), (1.0, (0.5, 0.5, 0.5))):
        for m in (0.0, 0.5, 1.0):
            check(vg(k, 0.5, (0, 0, 0)), vg(k + 1, vs_q, o_q), m)
            check(vg(k + 1, vs_q, o_q), vg(k, 0.5, (0, 0, 0)), m)
    recs = [OC.prim(OC.SPHERE, np.array([[1, 0, 0, x], [0, 1, 0, 0.25], [0, 0, 1, 0.25], [0, 0, 0, 1]]), radius=0.25)
            for x in (0.75, 1.0, 1.25, 1.5)]
    recs += [OC.prim(OC.BOX, np.array([[1, 0, 0, x], [0, 1, 0, 0.25], [0, 0, 1, 0.25], [0, 0, 0, 1]]), lengths=[0.5, 0.5, 0.5])
             for x in (0.75, 1.0, 1.25)]
    for m in (0.0, 0.25):
        check(vg([[0, 0, 0]], 0.5, (0, 0, 0)), prims(recs), m)
        check(prims(recs), vg([[0, 0, 0]], 0.5, (0, 0, 0)), m)


def test_occupancy_grid_after_insert_and_free_area():
    from cupoch_b200.testing import datagen
    pts, _ = datagen.surface(20000, 3)
    o = G.OccupancyGrid(0.05, 64, (0.0, 0.0, 0.0))
    o.insert(G.PointCloud(pts.astype(np.float32)), (0.0, 0.0, 2.0))
    rng = np.random.default_rng(5)
    q = vg(np.floor(pts[::7] / 0.04).astype(np.int32), 0.04, (0.01, 0.0, -0.02))
    p = prims(random_prims(rng, 300, 1.0, 0.05))
    for m in (0.0, 0.025, 0.15):
        a = (o, occ_operand(o))
        n_before = len(check(a, q, m))
        check(q, a, m)
        check(a, p, m)
        check(p, a, m)
    assert n_before > 0
    o.set_free_area((-0.3, -0.3, -0.3), (0.3, 0.3, 0.3))  # shrinks the bound box: occupied cells outside never collide
    a = (o, occ_operand(o))
    for m in (0.0, 0.15):
        assert len(check(a, q, m)) < n_before
        check(q, a, m)
        check(a, p, m)
        check(p, a, m)


def test_one_primitive_covering_many_cells():
    p, keys, vs = big_rotated_box_scene()
    g = vg(keys, vs, (0, 0, 0))
    got = check(g, prims([p]), 0.0)
    assert got.tolist() == [[len(keys) - 1, 0]]
    check(prims([p]), g, 0.0)


def test_many_primitives():
    rng = np.random.default_rng(11)
    recs = random_prims(rng, 10_000, 2.0, 0.02)
    p = prims(recs)
    g = vg(cluster_keys(rng, 1000, 100), 0.02, (0.003, 0.001, -0.002))
    for m in (0.0, 0.01, 0.06):
        check(g, p, m)
        check(p, g, m)


def test_2m_voxels_sampled_against_brute_force():
    rng = np.random.default_rng(13)
    keys = np.unique(cluster_keys(rng, 2_600_000, 400), axis=0)
    rng.shuffle(keys)
    assert len(keys) > 2_000_000
    vs = 0.02
    tgt, _ = vg(keys, vs, (0, 0, 0))
    qkeys = keys[rng.permutation(len(keys))]
    qry, _ = vg(qkeys, vs, (0.3 * vs, 0.2 * vs, 0.1 * vs))
    for m in (0.0, 2 * vs):
        pairs = K.compute_intersection(tgt, qry, m).get_collision_index_pairs()
        best = np.full(len(qkeys), -1, np.int64)
        best[pairs[:, 1]] = pairs[:, 0]
        for j in rng.choice(len(qkeys), 300, replace=False):
            near = np.flatnonzero(np.all(np.abs(keys - qkeys[j]) <= 4, 1))
            t = OC.voxel_grid(keys[near], vs, (0, 0, 0))
            b = OC.best(t, OC.voxel_grid(qkeys[j:j + 1], vs, (0.3 * vs, 0.2 * vs, 0.1 * vs)), m)[0]
            assert best[j] == (near[b] if b >= 0 else -1)


def test_launch_count_is_fixed_and_repeats_are_identical():
    L = _lib.lib()
    rng = np.random.default_rng(17)
    deltas = {}
    for n in (1000, 200_000):
        a, b = make("vg", n, rng, VS_T, O_T), make("vg", n, rng, VS_Q, O_Q)
        o = make("occ", min(n, 5000), rng, VS_T, O_T)
        p = make("prim", 100, rng, VS_T, O_T)
        for name, x, y in (("vg_vg", a, b), ("vg_occ", a, o), ("occ_vg", o, b), ("vg_prim", a, p), ("prim_vg", p, a),
                           ("occ_prim", o, p), ("prim_occ", p, o)):
            first = K.compute_intersection(x[0], y[0], 0.3).get_collision_index_pairs()
            assert len(first), name
            c0 = L.cphb_launch_count()
            again = K.compute_intersection(x[0], y[0], 0.3).get_collision_index_pairs()
            deltas.setdefault(name, set()).add(L.cphb_launch_count() - c0)
            assert np.array_equal(first, again)
    for name, d in deltas.items():
        assert len(d) == 1, (name, d)


def test_illegal_arguments(capfd):
    g, _ = vg([[0, 0, 0]], 1.0, (0, 0, 0))
    s = K.PrimitiveArray([K.Sphere(1.0)])
    for m in (float("nan"), float("inf")):
        assert not K.compute_intersection(g, g, m).is_collided()
    for vs in (0.0, -1.0, float("nan"), float("inf")):
        bad, _ = vg([[0, 0, 0]], 1.0, (0, 0, 0))
        bad.voxel_size = vs
        assert not K.compute_intersection(bad, g).is_collided()
        assert not K.compute_intersection(g, bad).is_collided()
    o = G.OccupancyGrid(1.0, 8)
    o.add_voxels(np.array([[4, 4, 4]], np.int32), True)
    o.voxel_size = 0.0
    assert not K.compute_intersection(o, g).is_collided()
    wide, _ = vg([[0, 0, 0], [1 << 21, 0, 0]], 1.0, (0, 0, 0))
    assert not K.compute_intersection(wide, g).is_collided()
    ok, _ = vg([[0, 0, 0], [(1 << 21) - 1, 0, 0]], 1.0, (0, 0, 0))
    assert K.compute_intersection(ok, g).is_collided()
    assert "[cupoch_b200][error]" in capfd.readouterr().err
    with pytest.raises(TypeError):
        K.compute_intersection(s, s)
    with pytest.raises(TypeError):
        K.compute_intersection(o, o)
    L = _lib.lib()
    cnt = C.c_size_t(7)
    occ = _lib.CollOperand(kind=K.CollisionType.OccupancyGrid, occ=o._h.value)
    pr = _lib.CollOperand(kind=K.CollisionType.Primitives)
    assert L.cphb_compute_intersection(C.byref(occ), C.byref(occ), 0.0, None, 0, C.byref(cnt), None) == _lib.CPHB_ERR_INVALID
    assert L.cphb_compute_intersection(C.byref(pr), C.byref(pr), 0.0, None, 0, C.byref(cnt), None) == _lib.CPHB_ERR_INVALID
    assert L.cphb_compute_intersection(None, C.byref(pr), 0.0, None, 0, C.byref(cnt), None) == _lib.CPHB_ERR_INVALID


def test_empty_operands_warn(capfd):
    g, _ = vg([[0, 0, 0]], 1.0, (0, 0, 0))
    e, _ = vg(np.zeros((0, 3), np.int32), 1.0, (0, 0, 0))
    assert not K.compute_intersection(g, e).is_collided()
    assert not K.compute_intersection(K.PrimitiveArray(), g).is_collided()
    assert "target or query is empty" in capfd.readouterr().err
