"""CPU: oracle/mesh_ops.c -- TriangleMesh's ComputeEdgeList, the four vertex filters, GetSurfaceArea and
SamplePointsUniformly -- against the reference's googletest fixtures (tests/golden/mesh_ops_known.json), a numpy edge
list, a float64 restatement of every filter pass, and the geometry and statistics of uniform sampling."""
import json
import os

import numpy as np
import pytest
from scipy import stats

from oracle import mesh_ops_py as M

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mesh_ops_known.json")
EPS32 = 2.0 ** -24


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def random_mesh(seed, nv=300, nt=500, isolated=(7, 150), repeat=True, duplicate=True):
    """random triangles over nv vertices, none using the `isolated` ones; one triangle with a repeated vertex and two
    vertices at the same position (a zero-length edge)"""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(nv, 3)).astype(np.float32)
    pool = np.setdiff1d(np.arange(nv), isolated)
    t = np.stack([rng.choice(pool, 3, replace=False) for _ in range(nt)]).astype(np.int32)
    if repeat:
        t[3] = (t[3, 0], t[3, 0], t[3, 2])
    if duplicate:
        v[t[5, 1]] = v[t[5, 0]]
    n = rng.normal(size=(nv, 3)).astype(np.float32)
    c = rng.uniform(0, 1, (nv, 3)).astype(np.float32)
    return v, t, n, c


def numpy_edges(t):
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 0]], t[:, [1, 2]], t[:, [2, 1]], t[:, [2, 0]], t[:, [0, 2]]]).astype(np.int64)
    return np.unique(e, axis=0).astype(np.int32)


def test_golden_edge_list():
    g = golden()["edge_list"]
    assert np.array_equal(M.edge_list(g["triangles"], len(g["vertices"])), np.int32(g["edges"]))


def test_golden_filters_within_the_reference_tolerance():
    g = golden()
    f = g["filters"]
    v0 = np.float32(f["vertices"])
    e = M.edge_list(f["triangles"], len(v0))
    cur = {}
    for st in f["steps"]:
        k, a = st["filter"], st["args"]
        v = cur.get(k, v0)
        it = a["number_of_iterations"]
        out = {"sharpen": lambda: M.sharpen(e, v, iterations=it, strength=a["strength"]),
               "simple": lambda: M.smooth_simple(e, v, iterations=it),
               "laplacian": lambda: M.smooth_laplacian(e, v, iterations=it, lambda_=a["lambda"]),
               "taubin": lambda: M.smooth_taubin(e, v, iterations=it, lambda_=a["lambda"], mu=a["mu"])}[k]()[0]
        np.testing.assert_allclose(out, np.float32(st["vertices"]), rtol=0, atol=g["tolerance"], err_msg=str(st))
        cur[k] = out


def test_golden_sampling_counts_and_attributes():
    s = golden()["sample_points_uniformly"]
    n = s["number_of_points"]
    for case in s["cases"]:
        kw = {a: s[a] for a in case["attributes"]}
        tn = None
        if case["use_triangle_normal"]:
            tn = np.float32([[0, 0, 1]])  # the normalised triangle normal of (0,0,0), (1,0,0), (0,1,0)
        p, nr, c, _ = M.sample_points_uniformly(s["vertices"], s["triangles"], n, triangle_normals=tn, **kw)
        assert len(p) == case["points"]
        assert (0 if nr is None else len(nr)) == case["normals"] and (0 if c is None else len(c)) == case["colors"]
        if c is not None:
            np.testing.assert_allclose(c, np.float32([case["color"]] * n), atol=1e-4)
        if nr is not None:
            np.testing.assert_allclose(nr, np.float32([case["normal"]] * n), atol=1e-4)
    with pytest.raises(ValueError):
        M.sample_points_uniformly(np.zeros((0, 3)), np.zeros((0, 3), np.int32), 100)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_edge_list_is_the_unique_directed_edges(seed):
    v, t, _, _ = random_mesh(seed)
    e = M.edge_list(t, len(v))
    assert np.array_equal(e, numpy_edges(t))
    assert [t[3, 0], t[3, 0]] in e.tolist()  # the repeated vertex's self-edge is kept, as the reference keeps it


def test_edge_list_rejects_an_index_out_of_range():
    with pytest.raises(ValueError):
        M.edge_list(np.int32([[0, 1, 3]]), 3)
    with pytest.raises(ValueError):
        M.edge_list(np.int32([[0, -1, 2]]), 3)


def pass64(kind, c, e, prev, v_in):
    """one pass in float64 over explicit neighbour lists -> (result, magnitude bound for the float32 error)"""
    nv = len(prev)
    out, mag = prev.astype(np.float64).copy(), np.zeros((nv, 3))
    rows = {}
    for a, b in e:
        rows.setdefault(int(a), []).append(int(b))
    p = prev.astype(np.float64)
    for vtx, nb in rows.items():
        N = len(nb)
        x = p[nb]
        if kind == M.SHARPEN:
            s = x.sum(0)
            out[vtx] = p[vtx] + c * (p[vtx] * N - s)
            mag[vtx] = np.abs(p[vtx]) + abs(c) * (np.abs(p[vtx]) * N + np.abs(x).sum(0)) * (N + 2)
        elif kind == M.SIMPLE:
            out[vtx] = (p[vtx] + x.sum(0)) / (1.0 + N)
            mag[vtx] = (np.abs(p[vtx]) + np.abs(x).sum(0)) / (1.0 + N) * (N + 2)
        else:
            d = np.linalg.norm(v_in[vtx].astype(np.float64) - v_in[nb].astype(np.float64), axis=1)
            d32 = np.sqrt(((v_in[vtx] - v_in[nb]).astype(np.float32) ** 2).sum(1, dtype=np.float32))
            w = (1.0 / (d32.astype(np.float64) + 1e-12)).astype(np.float32).astype(np.float64)  # the weights' own rounding
            assert np.all(np.abs(d32 - d) <= 4 * EPS32 * np.maximum(d, 1e-30) + 1e-30)
            s = (w[:, None] * x).sum(0) / w.sum()
            out[vtx] = p[vtx] + c * (s - p[vtx])
            mag[vtx] = np.abs(p[vtx]) + abs(c) * (np.abs(x).max(0) * (N + 3) + np.abs(p[vtx]))
    return out, mag


@pytest.mark.parametrize("kind,c", [(M.SHARPEN, 0.3), (M.SIMPLE, 0.0), (M.LAPLACIAN, 0.5), (M.LAPLACIAN, -0.53)])
@pytest.mark.parametrize("seed", [3, 4])
def test_each_filter_pass_is_within_a_few_ulps_of_float64(kind, c, seed):
    v, t, n, col = random_mesh(seed)
    e = M.edge_list(t, len(v))
    cur = [v, n, col]
    for _ in range(3):  # pass by pass: each from the oracle's own previous float32 result
        nxt = M.filter_mesh(kind, 1, e, *cur, mask=7, c0=c)
        for a in range(3):
            want, mag = pass64(kind, c, e, cur[a], v)
            err = np.abs(nxt[a].astype(np.float64) - want)
            assert np.all(err <= 4 * EPS32 * mag + 1e-38), (a, float((err / np.maximum(mag, 1e-30)).max() / EPS32))
        cur = [nxt[0] if kind < M.LAPLACIAN else v, nxt[1], nxt[2]]  # Laplacian weights stay those of the input vertices


def test_isolated_vertices_and_degenerate_triangles_keep_the_rows_aligned():
    v, t, n, c = random_mesh(9)
    e = M.edge_list(t, len(v))
    for kind in (M.SHARPEN, M.SIMPLE, M.LAPLACIAN, M.TAUBIN):
        out = M.filter_mesh(kind, 5, e, v, n, c, mask=7, c0=0.3, c1=-0.31)
        for a, src in zip(out, (v, n, c)):
            assert np.array_equal(a[[7, 150]], src[[7, 150]])  # no neighbours: unchanged
            assert np.all(np.isfinite(a))  # the zero-length edge's weight is 1e12, finite
    # one pass of Simple at a vertex next to the isolated one reads its own neighbours only
    out = M.smooth_simple(e, v, iterations=1)[0]
    want, _ = pass64(M.SIMPLE, 0.0, e, v, v)
    np.testing.assert_allclose(out, want, rtol=1e-5, atol=1e-6)


def test_scope_iterations_zero_and_bad_edge_lists():
    v, t, n, c = random_mesh(11)
    e = M.edge_list(t, len(v))
    for mask, moved in ((1, (0,)), (2, (1,)), (4, (2,)), (7, (0, 1, 2))):
        out = M.sharpen(e, v, n, c, iterations=2, strength=0.1, mask=mask)
        for a, src in enumerate((v, n, c)):
            assert np.array_equal(out[a], src) != (a in moved)
    out = M.smooth_taubin(e, v, n, c, iterations=0)
    assert all(np.array_equal(a, b) for a, b in zip(out, (v, n, c)))
    with pytest.raises(ValueError):
        M.smooth_simple(e[::-1], v)
    bad = e.copy()
    bad[-1, 1] = len(v)
    with pytest.raises(ValueError):
        M.smooth_simple(bad, v)


def test_surface_area_is_the_float64_sum():
    v, t, _, _ = random_mesh(12, nv=2000, nt=400000)
    total, areas = M.surface_area(v, t)
    p0, p1, p2 = (v[t[:, k]].astype(np.float64) for k in range(3))
    a64 = 0.5 * np.linalg.norm(np.cross(p0 - p1, p0 - p2), axis=1)
    scale = np.maximum(np.abs(p0 - p1).max(1), np.abs(p0 - p2).max(1)) ** 2  # the cross product's cancellation
    assert np.all(np.abs(areas - a64) <= 8 * EPS32 * (a64 + scale))
    assert total == np.float32(areas.astype(np.float64).sum())  # any float64 order rounds to the same float here


def test_sampling_gives_exactly_n_points_inside_their_triangles():
    v, t, vn, vc = random_mesh(13, nv=400, nt=700)
    _, areas = M.surface_area(v, t)
    for n in (1, 699, 700, 701, 50000):
        p, nr, c, b = M.sample_points_uniformly(v, t, n, vertex_normals=vn, vertex_colors=vc)
        assert len(p) == n and b[0] == 0 and b[-1] == n and np.all(np.diff(b.astype(np.int64)) >= 0)
        cnt = np.diff(b.astype(np.int64))
        want = n * areas.astype(np.float64) / areas.astype(np.float64).sum()
        assert np.all(np.abs(cnt - want) <= 1.0 + 1e-9)
        tri = np.repeat(np.arange(len(t)), cnt)
        P = v[t[tri]].astype(np.float64)
        # barycentric coordinates of each point in its own triangle
        e0, e1, q = P[:, 1] - P[:, 0], P[:, 2] - P[:, 0], p.astype(np.float64) - P[:, 0]
        d00, d01, d11 = (e0 * e0).sum(1), (e0 * e1).sum(1), (e1 * e1).sum(1)
        d20, d21 = (q * e0).sum(1), (q * e1).sum(1)
        den = d00 * d11 - d01 * d01
        ok = den > 1e-12
        bb = (d11 * d20 - d01 * d21)[ok] / den[ok]
        cc = (d00 * d21 - d01 * d20)[ok] / den[ok]
        assert np.all(bb >= -1e-5) and np.all(cc >= -1e-5) and np.all(bb + cc <= 1 + 1e-5)


def test_sampling_is_uniform_chi_square():
    # equal-area triangles get n / nt points each; inside a triangle the four midpoint sub-triangles are equally likely
    v = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [2, 0, 0], [2, 1, 0]])
    t = np.int32([[0, 1, 2], [1, 3, 2], [1, 4, 3], [4, 5, 3]])
    n = 40000
    p, _, _, b = M.sample_points_uniformly(v, t, n)
    cnt = np.diff(b.astype(np.int64))
    assert stats.chisquare(cnt).pvalue > 0.01 and cnt.sum() == n
    P = v[t[0]].astype(np.float64)
    q = p[:cnt[0]].astype(np.float64)
    x, y = q[:, 0], q[:, 1]  # triangle 0 is the unit right triangle: sub-triangles by x < 1/2, y < 1/2
    cell = np.where(x >= 0.5, 0, np.where(y >= 0.5, 1, np.where(x + y <= 0.5, 2, 3)))
    assert P[0].tolist() == [0, 0, 0]
    assert stats.chisquare(np.bincount(cell, minlength=4)).pvalue > 0.001


def test_sampling_rejects_zero_area_and_bad_arguments():
    v = np.float32([[0, 0, 0], [1, 0, 0], [2, 0, 0]])
    with pytest.raises(ValueError):
        M.sample_points_uniformly(v, np.int32([[0, 1, 2]]), 10)
    with pytest.raises(ValueError):
        M.sample_points_uniformly(v, np.int32([[0, 1, 3]]), 10)
    with pytest.raises(ValueError):
        M.sample_points_uniformly(np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]]), np.int32([[0, 1, 2]]), 0)
