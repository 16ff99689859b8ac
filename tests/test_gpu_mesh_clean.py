"""GPU: TriangleMesh cleanup, + / +=, and get_self_intersecting_triangles (csrc/mesh_clean.cu) against
oracle/mesh_clean.c bit for bit: random meshes with quantised coordinates (many duplicates, -0 / +0, NaN and inf), every
combination of vertex normals, colours and triangle normals with and without an edge list, empty and triangle-less
meshes; the weld round trip of TSDF sphere meshes; self-intersections of random soups, two overlapping spheres joined
with +=, an un-welded soup before and after welding, coplanar grids, 2000 coincident triangles, one huge triangle among
small ones, tiny triangles over a 1e6 extent and non-finite vertices.  Also the sizing / writing calls, repeats, the
launch count and every rejection."""
import itertools

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import mesh_clean_py as MC

G, CAM, I = cph.geometry, cph.camera, cph.integration
CT = I.TSDFVolumeColorType


def sphere_mesh(res=128, views=8, centre=(0.0, 0.0, 0.0)):
    """test_gpu_mesh_ops.py's recipe: a radius-0.6 sphere seen from a ring of cameras, fused into a 2 m volume"""
    w, h = 160, 120
    vol = I.UniformTSDFVolume(2.0, res, 0.06, CT.RGB8)
    rng = np.random.default_rng(res)
    for K, E in ring_cameras(views, w, h, 2.5):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)), G.Image(d16),
                                                     1000.0, 100.0, False)
        vol.integrate(im, CAM.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    m = vol.extract_triangle_mesh()
    if any(centre):
        out = G.TriangleMesh(m.vertices.cpu() + np.asarray(centre, np.float32), m.triangles.cpu())
        return out
    return m


def quantised_mesh(seed, nv=3000, nt=4000, q=4):
    rng = np.random.default_rng(seed)
    v = (rng.integers(-q, q + 1, (nv, 3)) / np.float32(q)).astype(np.float32)
    v[rng.random(nv) < 0.05] *= np.float32(-1)  # makes -0 from +0
    v[7] = (np.nan, 0, 0)
    v[11] = (0, np.nan, 1)
    v[13] = (np.inf, 0, 0)
    v[17] = (-np.inf, 0, 0)
    t = rng.integers(0, nv, (nt, 3)).astype(np.int32)
    t[::9, 2] = t[::9, 0]
    t[5::13] = t[4::13][: len(t[5::13])]  # duplicates
    t[6::17] = t[4::17][: len(t[6::17])][:, [1, 2, 0]]  # rotated duplicates
    return v, t


def build_mesh(v, t, vn, vc, tn, el):
    rng = np.random.default_rng(len(v))
    m = G.TriangleMesh(v, t)
    if vn:
        m.vertex_normals = rng.normal(size=(len(v), 3)).astype(np.float32)
    if vc:
        m.vertex_colors = rng.random((len(v), 3)).astype(np.float32)
    if tn:
        m.triangle_normals = rng.normal(size=(len(t), 3)).astype(np.float32)
    if el:
        m.compute_edge_list()
    return m


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                                 b.view(np.uint32) if b.dtype == np.float32 else b)


def cpu(a):
    return None if a is None else a.cpu()


COMBOS = list(itertools.product([False, True], repeat=4))


@pytest.mark.parametrize("vn,vc,tn,el", COMBOS)
def test_remove_ops_match_the_oracle(vn, vc, tn, el):
    v, t = quantised_mesh(1)
    m = build_mesh(v, t, vn, vc, tn, el)
    N, C, TN = cpu(m.vertex_normals), cpu(m.vertex_colors), cpu(m.triangle_normals)

    a = build_mesh(v, t, vn, vc, tn, el)
    a.vertex_normals, a.vertex_colors, a.triangle_normals = m.vertex_normals, m.vertex_colors, m.triangle_normals
    a.remove_duplicated_vertices()
    ov, ot, on, oc = MC.remove_duplicated_vertices(v, t, N, C)
    assert same(a.vertices.cpu(), ov) and same(a.triangles.cpu(), ot)
    assert (on is None) == (not vn) and (on is None or same(a.vertex_normals.cpu(), on))
    assert (oc is None) == (not vc) and (oc is None or same(a.vertex_colors.cpu(), oc))
    assert tn == a.has_triangle_normals() and (not tn or same(a.triangle_normals.cpu(), TN))
    if el:
        ref = G.TriangleMesh(ov, ot).compute_edge_list().edge_list.cpu()
        assert same(a.edge_list.cpu(), ref)

    # the triangle passes run on the welded mesh, so duplicates by index exist
    t2, tn2 = MC.remove_duplicated_triangles(ot, len(ov), TN)
    a.remove_duplicated_triangles()
    assert same(a.triangles.cpu(), t2) and (tn2 is None or same(a.triangle_normals.cpu(), tn2))
    t3, tn3 = MC.remove_degenerate_triangles(t2, len(ov), tn2)
    a.remove_degenerate_triangles()
    assert same(a.triangles.cpu(), t3) and (tn3 is None or same(a.triangle_normals.cpu(), tn3))
    v4, t4, n4, c4 = MC.remove_unreferenced_vertices(ov, t3, on, oc)
    a.remove_unreferenced_vertices()
    assert same(a.vertices.cpu(), v4) and same(a.triangles.cpu(), t4)
    assert n4 is None or same(a.vertex_normals.cpu(), n4)
    assert c4 is None or same(a.vertex_colors.cpu(), c4)
    if el:
        assert same(a.edge_list.cpu(), G.TriangleMesh(v4, t4).compute_edge_list().edge_list.cpu())


@pytest.mark.parametrize("vn,vc,tn,el", COMBOS)
def test_iadd_matches_the_oracle(vn, vc, tn, el):
    va, ta = quantised_mesh(2, 500, 700)
    vb, tb = quantised_mesh(3, 300, 400)
    a = build_mesh(va, ta, vn, vc, tn, el)
    b = build_mesh(vb, tb, True, vc, tn, False)
    c = a + b
    assert len(a.vertices) == 500  # + leaves its left side alone
    a += b
    for m in (a, c):
        assert same(m.vertices.cpu(), np.concatenate([va, vb]))
        assert same(m.triangles.cpu(), MC.append_triangles(ta, 500, tb, 300))
        assert m.has_vertex_normals() == vn and m.has_vertex_colors() == vc and m.has_triangle_normals() == tn
        if vn:
            assert same(m.vertex_normals.cpu()[500:], b.vertex_normals.cpu())
        assert m.has_edge_list() == el
    e = G.TriangleMesh()
    e += b
    assert e.has_vertex_normals() and same(e.triangles.cpu(), tb)
    n0 = len(a.triangles)
    a += G.TriangleMesh()
    assert len(a.triangles) == n0


def test_empty_and_triangle_less_meshes():
    for m in (G.TriangleMesh(), G.TriangleMesh(np.ones((5, 3), np.float32))):
        m.remove_duplicated_vertices().remove_duplicated_triangles().remove_degenerate_triangles()
        assert len(m.get_self_intersecting_triangles()) == 0
    m = G.TriangleMesh(np.ones((5, 3), np.float32))
    m.remove_duplicated_vertices()
    assert len(m.vertices) == 1
    m = G.TriangleMesh(np.ones((5, 3), np.float32))
    m.remove_unreferenced_vertices()
    assert len(m.vertices) == 0
    m = G.TriangleMesh(np.arange(9, dtype=np.float32).reshape(3, 3), np.array([[0, 0, 1], [2, 2, 2]], np.int32))
    m.remove_degenerate_triangles()
    assert len(m.triangles) == 0


@pytest.mark.parametrize("res", [128, 256])
def test_weld_round_trip(res):
    m = sphere_mesh(res)
    v, t = m.vertices.cpu(), m.triangles.cpu()
    soup = G.TriangleMesh(v[t.reshape(-1)], np.arange(3 * len(t), dtype=np.int32).reshape(-1, 3))
    soup.remove_duplicated_vertices()
    used = np.unique(t)
    ref = v[used][np.lexsort(v[used].T[::-1])]
    assert same(soup.vertices.cpu(), ref)
    assert same(soup.vertices.cpu()[soup.triangles.cpu()], v[t])


def check_self(m, mode=None):
    v, t = m.vertices.cpu(), m.triangles.cpu()
    got, cand = m._self_intersections()
    got = got.cpu()
    if mode is None:
        mode = MC.ALL_PAIRS if len(t) <= 3000 else MC.SWEEP
    ref = MC.self_intersections(v, t, mode, True)
    assert same(got, ref), (len(got), len(ref))
    assert cand >= len(ref)
    return got


def soup_mesh(seed, n, scale=1.0, size=0.2, shift=10.0):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-scale, scale, (n, 1, 3))
    v = (c + rng.normal(size=(n, 3, 3)) * size).reshape(-1, 3).astype(np.float32) + np.float32(shift)
    return G.TriangleMesh(v.astype(np.float32), np.arange(3 * n, dtype=np.int32).reshape(n, 3))


@pytest.mark.parametrize("seed,n", [(1, 500), (2, 3000), (3, 20000)])
def test_random_soups(seed, n):
    assert len(check_self(soup_mesh(seed, n, 1.0, 0.05))) > 0


def test_two_overlapping_spheres():
    a = sphere_mesh(128)
    b = sphere_mesh(128, centre=(0.3, 0.1, 0.0))
    u = a + b
    got = check_self(u)
    na = len(a.triangles)
    cross = (got[:, 0] < na) & (got[:, 1] >= na)
    assert cross.sum() > 0
    # the pairs inside each sphere are each sphere's own (marching cubes leaves a few touching pairs of its own)
    assert same(got[got[:, 1] < na], check_self(a))
    assert same(got[got[:, 0] >= na] - na, check_self(b))


def test_unwelded_soup_then_welded():
    m = sphere_mesh(64)
    v, t = m.vertices.cpu(), m.triangles.cpu()
    soup = G.TriangleMesh(v[t.reshape(-1)], np.arange(3 * len(t), dtype=np.int32).reshape(-1, 3))
    own = check_self(m)
    assert len(check_self(soup)) > len(t) + len(own)  # adjacent triangles touch and share no index
    soup.remove_duplicated_vertices()
    assert same(check_self(soup), own)  # welded, only the mesh's own pairs are left


def test_coplanar_grid():
    k = 40
    xs = np.arange(k, dtype=np.float32) * 0.5
    v, t = [], []
    for x in xs:
        for y in xs:
            b = len(v)
            v += [[x, y, 0], [x + 0.7, y, 0], [x, y + 0.7, 0]]
            t.append([b, b + 1, b + 2])
    assert len(check_self(G.TriangleMesh(np.array(v, np.float32), np.array(t, np.int32)))) > 0


def test_coincident_triangles():
    tri = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    n = 2000
    m = G.TriangleMesh(np.tile(tri, (n, 1)), np.arange(3 * n, dtype=np.int32).reshape(n, 3))
    got = m.get_self_intersecting_triangles().cpu()
    i, j = np.triu_indices(n, 1)
    assert len(got) == 1999000 and same(got, np.stack([i, j], 1).astype(np.int32))


def test_one_huge_triangle_among_small_ones():
    s = soup_mesh(4, 10000, 5.0, 0.02, 0.0)
    v = np.concatenate([s.vertices.cpu(), np.array([[-6, -6, 0], [6, -6, 0.1], [0, 6, -0.1]], np.float32)])
    t = np.concatenate([s.triangles.cpu(), [[30000, 30001, 30002]]]).astype(np.int32)
    got = check_self(G.TriangleMesh(v, t), MC.SWEEP)
    assert (got[:, 1] == 10000).sum() > 0


def test_tiny_triangles_over_a_huge_extent():
    s = soup_mesh(5, 5000, 5e5, 0.5, 0.0)
    v = s.vertices.cpu()
    v[:3] = [[-1e6, 0, 0], [-1e6 + 1, 0, 0], [-1e6, 1, 0]]
    v[3:6] = [[1e6, 0, 0], [1e6 + 1, 0, 0], [1e6, 1, 0]]
    v[6:9] = [[1e6, 0.2, -1], [1e6 + 0.2, 0.2, 1], [1e6 + 0.3, 0.3, 1]]
    assert len(check_self(G.TriangleMesh(v, s.triangles.cpu()), MC.SWEEP)) > 0


def test_non_finite_vertices():
    s = soup_mesh(6, 800, 0.5, 0.1)
    v = s.vertices.cpu()
    v[0] = (np.inf, 0, 0)
    v[4] = (np.nan, 1, 1)
    v[8] = (0, -np.inf, 0)
    got = check_self(G.TriangleMesh(v, s.triangles.cpu()))
    assert not np.isin(got, [0, 1, 2]).any()


def test_sizing_repeats_and_launch_count():
    m = soup_mesh(7, 3000, 1.0, 0.05)
    L = _lib.lib()
    n, c = ctypes_sizes(m)
    assert n > 0
    runs, launches = [], []
    for _ in range(3):
        n0 = L.cphb_launch_count()
        runs.append(m.get_self_intersecting_triangles().cpu())
        launches.append(L.cphb_launch_count() - n0)
    assert all(same(r, runs[0]) for r in runs) and len(runs[0]) == n
    other = soup_mesh(8, 500, 1.0, 0.05)
    n0 = L.cphb_launch_count()
    other.get_self_intersecting_triangles()
    assert len(set(launches)) == 1 and L.cphb_launch_count() - n0 == launches[0]


def ctypes_sizes(m):
    import ctypes as C
    cnt, cand = C.c_size_t(0), C.c_size_t(0)
    _lib.check(_lib.lib().cphb_mesh_self_intersecting_triangles(m.vertices.ptr, len(m.vertices), m.triangles.ptr, len(m.triangles), None, 0,
                                                                C.byref(cnt), C.byref(cand), None))
    return cnt.value, cand.value


def test_every_rejection_changes_nothing():
    v = np.zeros((4, 3), np.float32)
    for bad in ([[0, 1, 4]], [[-1, 1, 2]]):
        m = G.TriangleMesh(v, np.array(bad, np.int32))
        for op in (m.remove_duplicated_vertices, m.remove_duplicated_triangles, m.remove_unreferenced_vertices,
                   m.remove_degenerate_triangles, m.get_self_intersecting_triangles):
            with pytest.raises(_lib.CphbError):
                op()
            assert same(m.triangles.cpu(), np.array(bad, np.int32)) and len(m.vertices) == 4
        g = G.TriangleMesh(v, np.array([[0, 1, 2]], np.int32))
        with pytest.raises(_lib.CphbError):
            g += m
        assert len(g.vertices) == 4 and len(g.triangles) == 1
    # after the rejections the same mesh still cleans normally
    assert G.TriangleMesh(v, np.array([[0, 1, 2]], np.int32)).remove_duplicated_vertices().vertices.shape == (1, 3)


def test_golden_pairs_as_two_triangle_meshes():
    """every pair of tests/golden/tritri_ref.npz (the reference header's own answers) as a two-triangle mesh: the device
    reports it exactly when the reference does and the closed boxes overlap"""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tritri_ref.npz"))
    p, q, hit = g["p"], g["q"], g["hit"]
    t = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    for a, b, h in zip(p, q, hit):
        overlap = bool((a.min(0) <= b.max(0)).all() and (b.min(0) <= a.max(0)).all())
        got = G.TriangleMesh(np.concatenate([a, b]), t).get_self_intersecting_triangles().cpu()
        assert len(got) == int(bool(h) and overlap), (a, b, h)


def test_two_crossing_large_triangles_among_small_ones():
    """two triangles that each cover more than SI_K cells and cross each other: the pair is reported once (by the lower
    index's warp), and every pair equals the oracle's"""
    s = soup_mesh(9, 4000, 5.0, 0.02, 0.0)
    v = np.concatenate([s.vertices.cpu(), np.array([[-6, -6, 0], [6, -6, 0.1], [0, 6, -0.1],
                                                     [-6, 0, -3], [6, 0.5, 3], [0, -0.5, 3]], np.float32)])
    t = np.concatenate([s.triangles.cpu(), [[12000, 12001, 12002], [12003, 12004, 12005]]]).astype(np.int32)
    got = check_self(G.TriangleMesh(v, t), MC.SWEEP)
    assert ((got[:, 0] == 4000) & (got[:, 1] == 4001)).sum() == 1
    assert (got[:, 1] == 4000).sum() > 0  # the first also cuts small ones; the rest of both rows is held by the oracle


def test_capacity_too_small_writes_nothing():
    import ctypes as C
    m = soup_mesh(10, 600, 0.5, 0.1)
    n, _ = ctypes_sizes(m)
    assert n > 2
    buf = cph.utility.DeviceArray((n, 2), np.int32)
    sentinel = np.full((n, 2), -7, np.int32)
    _lib.check(_lib.lib().cphb_memcpy_h2d(buf.ptr, sentinel.ctypes.data, sentinel.nbytes, None))
    cnt = C.c_size_t(0)
    _lib.check(_lib.lib().cphb_mesh_self_intersecting_triangles(m.vertices.ptr, len(m.vertices), m.triangles.ptr, len(m.triangles), buf.ptr,
                                                                n - 1, C.byref(cnt), None, None))
    assert cnt.value == n and (buf.cpu() == -7).all()


def test_weld_round_trip_real_frames():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsdf_rgbd_known.npz"))
    K = CAM.PinholeCameraIntrinsic(CAM.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    vol = I.UniformTSDFVolume(8.0, 200, 0.04, CT.RGB8)
    rng = np.random.default_rng(5)
    for i in range(5):
        color = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(color), G.Image(g["depth"][i]), 1000.0, 4.0, False)
        vol.integrate(im, K, g["extrinsics"][i])
    m = vol.extract_triangle_mesh()
    v, t = m.vertices.cpu(), m.triangles.cpu()
    assert len(t) > 1000
    soup = G.TriangleMesh(v[t.reshape(-1)], np.arange(3 * len(t), dtype=np.int32).reshape(-1, 3))
    soup.remove_duplicated_vertices()
    ov, ot, _, _ = MC.remove_duplicated_vertices(v[t.reshape(-1)], np.arange(3 * len(t), dtype=np.int32).reshape(-1, 3))
    assert same(soup.vertices.cpu(), ov) and same(soup.triangles.cpu(), ot)
    assert same(soup.vertices.cpu()[soup.triangles.cpu()], v[t])


def test_edge_list_kept_when_nothing_is_removed():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], np.float32)
    m = G.TriangleMesh(v, np.array([[0, 1, 2], [1, 3, 2]], np.int32))
    m.edge_list = np.array([[0, 1]], np.int32)  # not the mesh's own: a recomputation would replace it
    for op in ("remove_duplicated_triangles", "remove_degenerate_triangles", "remove_unreferenced_vertices"):
        getattr(m, op)()
        assert same(m.edge_list.cpu(), [[0, 1]]), op
    m.remove_duplicated_vertices()  # recomputes whenever there is an edge list
    assert len(m.edge_list) == 10


def test_iadd_drops_what_the_right_hand_mesh_lacks():
    va, ta = quantised_mesh(11, 200, 300)
    vb, tb = quantised_mesh(12, 100, 150)
    a = build_mesh(va, ta, True, True, True, False)
    b = G.TriangleMesh(vb, tb)
    a += b
    assert not a.has_vertex_normals() and not a.has_vertex_colors() and not a.has_triangle_normals()
    assert len(a.vertices) == 300 and len(a.triangles) == 450


def test_remove_ops_launch_counts_are_fixed():
    L = _lib.lib()
    counts = {}
    for seed in (13, 14):
        v, t = quantised_mesh(seed, 2000 + 500 * seed, 3000 + 700 * seed)
        for op in ("remove_duplicated_vertices", "remove_duplicated_triangles", "remove_degenerate_triangles",
                   "remove_unreferenced_vertices"):
            m = G.TriangleMesh(v, t)
            n0 = L.cphb_launch_count()
            getattr(m, op)()
            counts.setdefault(op, set()).add(L.cphb_launch_count() - n0)
    assert all(len(c) == 1 for c in counts.values()), counts
