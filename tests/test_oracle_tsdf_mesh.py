"""CPU: the marching-cubes tables of tools/gen_mc_tables.py and the ExtractTriangleMesh / mesh-normal restatement
(oracle/tsdf_mesh.c) that the GPU tests hold the kernels to.

- The tables: the printed text is the text in csrc/tsdf.cu and oracle/tsdf_mesh.c; the edge table is the sign rule;
  every configuration's triangles draw exactly the face rule's segments on each face; complementary configurations
  draw the same segments reversed on every face that is not ambiguous.
- The reference's five real frames: 3198 vertices and 4402 triangles, cube by cube against the classic table.
- Closed analytic surfaces (sphere, torus, two spheres almost touching) give closed, consistently oriented
  2-manifolds with outward normals and vertices near the surface; random fields have no cracks between valid cubes.
- A float64 restatement of the vertex formula, the vertex-normal sum order, unreferenced vertices, NoColor and the
  int32 vertex limit."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_mc_tables as G  # noqa: E402
from oracle import tsdf_mesh_py as M, tsdf_py as T  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "tsdf_rgbd_known.npz")


def _block(path):
    with open(os.path.join(ROOT, path)) as f:
        s = f.read()
    return s[s.index(G.BEGIN):s.index(G.END) + len(G.END)] + "\n"


# ------------------------------------------------------------------------------------------------ the tables
def test_printed_tables_are_the_text_in_both_sources():
    text = G.c_block()
    assert _block("cupoch_b200/csrc/tsdf.cu") == text
    assert _block("oracle/tsdf_mesh.c") == text


def test_compiled_tables_are_the_generated_ones():
    e, c, t = M.tables()
    assert t.shape[1] == 3 * G.max_tris()
    for ci in range(256):
        tris = [x for tri in G.triangles(ci) for x in tri]
        assert e[ci] == G.edge_table(ci) and c[ci] == len(G.triangles(ci))
        assert list(t[ci, :len(tris)]) == tris and np.all(t[ci, len(tris):] == -1)


def test_edge_table_is_the_sign_rule():
    for ci in range(256):
        want = 0
        for e, (x, y, z, a) in enumerate(G.EDGE):
            o = (x, y, z)
            t = list(o)
            t[a] += 1
            if (ci >> G.CORNER.index(o) & 1) != (ci >> G.CORNER.index(tuple(t)) & 1):
                want |= 1 << e
        assert G.edge_table(ci) == want, ci


def _corners(e):
    x, y, z, a = G.EDGE[e]
    t = [x, y, z]
    t[a] += 1
    return G.CORNER.index((x, y, z)), G.CORNER.index(tuple(t))


def _faces():
    """(corners in cyclic order, outward normal) of the six faces, written independently of the generator"""
    out = []
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        for s in (0, 1):
            ring = []
            for u, v in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[a], p[b], p[c] = s, u, v
                ring.append(G.CORNER.index(tuple(p)))
            n = np.zeros(3)
            n[a] = 2 * s - 1
            out.append((ring, n))
    return out


def _edge_between(i, j):
    return next(e for e in range(12) if set(_corners(e)) == {i, j})


def _mid(e):
    i, j = _corners(e)
    return (np.array(G.CORNER[i]) + np.array(G.CORNER[j])) / 2.0


def _rule(ci, ring, n):
    """the face rule, restated: directed segments (a, b) on a face -- one for two crossed edges, one cutting off each
    negative corner on an ambiguous face -- running along g x n, g from the negative side to the positive side"""
    neg = [ci >> c & 1 for c in ring]
    sides = [_edge_between(ring[k], ring[(k + 1) % 4]) for k in range(4)]
    crossed = [sides[k] for k in range(4) if neg[k] != neg[(k + 1) % 4]]
    P = [np.array(G.CORNER[c], float) for c in ring]
    segs = []
    if len(crossed) == 2:
        g = np.mean([P[k] for k in range(4) if not neg[k]], 0) - np.mean([P[k] for k in range(4) if neg[k]], 0)
        segs.append((crossed[0], crossed[1], g))
    elif len(crossed) == 4:
        for k in range(4):
            if neg[k]:
                segs.append((sides[(k - 1) % 4], sides[k], np.mean(P, 0) - P[k]))
    out = set()
    for a, b, g in segs:
        out.add((a, b) if np.dot(_mid(b) - _mid(a), np.cross(g, n)) > 0 else (b, a))
    return out


def _boundary(tris):
    """the directed edges of a triangle set that are not cancelled by their reverse"""
    d = [(t[k], t[(k + 1) % 3]) for t in tris for k in range(3)]
    s = set(d)
    assert len(s) == len(d)
    return {e for e in s if (e[1], e[0]) not in s}


def test_triangles_draw_the_face_rule_on_every_face():
    for ci in range(256):
        bnd = _boundary(G.triangles(ci))
        want = set()
        for ring, n in _faces():
            segs = _rule(ci, ring, n)
            assert {s for s in bnd if all(set(_corners(e)) <= set(ring) for e in s)} == segs, (ci, ring)
            want |= segs
        assert bnd == want, ci


def test_complementary_configurations_draw_reversed_segments():
    for ci in range(256):
        for ring, n in _faces():
            neg = [ci >> c & 1 for c in ring]
            if neg[0] == neg[2] and neg[1] == neg[3] and neg[0] != neg[1]:
                continue  # ambiguous: the rule keeps the negative corners apart, which the complement swaps
            assert _rule(255 - ci, ring, n) == {(b, a) for a, b in _rule(ci, ring, n)}
        same = {tuple(p) for p in G.polygons(255 - ci)} == {tuple([p[0]] + p[1:][::-1]) for p in G.polygons(ci)}
        assert same or any(len([e for e in G.face_edges(r) if G.edge_table(ci) >> e & 1]) == 4 for r, _ in G.faces())


def test_max_triangle_count_is_reported():
    assert G.max_tris() == max(len(G.triangles(ci)) for ci in range(256)) == 5


# ------------------------------------------------------------------------------------------------ real frames
def _cube_indices(vol):
    r = vol.res
    f = vol.tw[:, 0].reshape(r, r, r)
    w = vol.tw[:, 1].reshape(r, r, r)
    ci = np.zeros((r - 1,) * 3, np.int32)
    valid = np.ones((r - 1,) * 3, bool)
    for i, (a, b, c) in enumerate(G.CORNER):
        valid &= w[a:a + r - 1, b:b + r - 1, c:c + r - 1] != 0
        ci |= (f[a:a + r - 1, b:b + r - 1, c:c + r - 1] < 0).astype(np.int32) << i
    return ci, valid


def _ambiguous(ci):
    return any(len([e for e in G.face_edges(r) if G.edge_table(ci) >> e & 1]) == 4 for r, _ in G.faces())


# the classic table's triangle counts for the configurations of the five cubes with an ambiguous face (cube (x, y, z):
# (configuration, classic count))
CLASSIC_AMBIGUOUS = {(152, 146, 135): (80, 2), (165, 158, 141): (104, 3), (166, 147, 128): (36, 2), (166, 156, 127): (66, 2),
                     (166, 157, 128): (66, 2)}


@pytest.fixture(scope="module")
def real_volume():
    g = np.load(GOLDEN)
    K = np.float32([[525, 0, 319.5], [0, 525, 239.5], [0, 0, 1]])
    vol = T.Volume(8.0, 200, 0.04, T.NO_COLOR)
    for i in range(5):
        vol.integrate(T.depth_to_float(g["depth"][i], 1000.0, 4.0), None, K, g["extrinsics"][i])
    return vol


def test_real_frames_give_3198_vertices_and_the_classic_triangle_count(real_volume):
    v, c, t = M.extract_triangle_mesh(real_volume)
    assert len(v) == 3198 and c is None
    ci, valid = _cube_indices(real_volume)
    emit = valid & (ci > 0) & (ci < 255)
    assert emit.sum() == 2197
    count = np.array([len(G.triangles(k)) for k in range(256)])
    amb = {tuple(int(x) for x in k): int(ci[tuple(k)]) for k in np.argwhere(emit) if _ambiguous(int(ci[tuple(k)]))}
    assert set(amb) == set(CLASSIC_AMBIGUOUS) and all(CLASSIC_AMBIGUOUS[k][0] == amb[k] for k in amb)
    # outside the ambiguous cubes every polygon is forced, and a table without extra vertices triangulates a
    # configuration with E crossed edges in P polygons with E - 2 P triangles, as the classic table does
    for k in np.unique(ci[emit]):
        if not _ambiguous(int(k)):
            assert count[k] == bin(G.edge_table(int(k))).count("1") - 2 * len(G.polygons(int(k)))
    ours_amb = sum(count[a] for a in amb.values())
    classic = count[ci[emit]].sum() - ours_amb + sum(n for _, n in CLASSIC_AMBIGUOUS.values())
    assert classic == 4402
    # pinned: the five ambiguous cubes get as many triangles here as under the classic table, so the total is 4402
    assert len(t) == 4402 and len(t) - classic == 0 and ours_amb == 11


# ------------------------------------------------------------------------------------------------ closed surfaces
def _field_volume(sdf, res=40, length=2.0, trunc=0.15, ct=T.NO_COLOR, seed=0):
    vol = T.Volume(length, res, trunc, ct)
    vl = vol.voxel_length
    k = (np.arange(res) - res // 2).astype(np.float64) * vl + vl / 2
    X, Y, Z = np.meshgrid(k, k, k, indexing="ij")
    vol.tw[:, 0] = np.clip(sdf(X, Y, Z) / trunc, -1, 1).astype(np.float32).reshape(-1)
    vol.tw[:, 1] = 1.0
    if ct != T.NO_COLOR:
        vol.col[:] = np.random.default_rng(seed).uniform(0, 255, vol.col.shape).astype(np.float32)
    return vol


def _sphere(c, r):
    return lambda X, Y, Z: np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r


def _torus(R, r):
    return lambda X, Y, Z: np.sqrt((np.sqrt(X ** 2 + Y ** 2) - R) ** 2 + Z ** 2) - r


def _two_spheres(gap):
    """two spheres of radius 0.35 a gap apart along the face diagonal (1, 1, 0): where they almost touch, voxels of
    the two spheres meet across the diagonals of cube faces"""
    d = np.array([1.0, 1.0, 0.0]) / np.sqrt(2)
    c = np.array([0.013, 0.011, 0.021])
    a, b = _sphere(c - (0.35 + gap / 2) * d, 0.35), _sphere(c + (0.35 + gap / 2) * d, 0.35)
    return lambda X, Y, Z: np.minimum(a(X, Y, Z), b(X, Y, Z))


def _directed_edges(t):
    return np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])


def _assert_closed_oriented_manifold(t):
    d = _directed_edges(t)
    keys = {(int(a), int(b)) for a, b in d}
    assert len(keys) == len(d), "a directed edge is used twice: inconsistent orientation"
    assert all((b, a) in keys for a, b in keys), "an edge is used once: the surface has a hole"
    return len(keys) // 2


@pytest.mark.parametrize("name,sdf,euler", [("sphere", _sphere((0.013, -0.027, 0.031), 0.6), 2),
                                            ("torus", _torus(0.55, 0.2), 0),
                                            ("two_spheres", _two_spheres(0.03), None)])
def test_closed_surfaces_are_oriented_manifolds(name, sdf, euler):
    vol = _field_volume(sdf)
    v, _, t = M.extract_triangle_mesh(vol)
    n_edges = _assert_closed_oriented_manifold(t)
    if euler is not None:
        assert len(v) - n_edges + len(t) == euler
    else:  # the two spheres meet in cubes with an ambiguous face
        ci, valid = _cube_indices(vol)
        assert sum(_ambiguous(int(k)) for k in ci[valid & (ci > 0) & (ci < 255)]) >= 2
    vd = v.astype(np.float64)
    n = np.cross(vd[t[:, 1]] - vd[t[:, 0]], vd[t[:, 2]] - vd[t[:, 0]])
    cen = vd[t].mean(1)
    h = 1e-5
    grad = np.stack([(sdf(*(cen + h * e).T) - sdf(*(cen - h * e).T)) / (2 * h) for e in np.eye(3)], 1)
    dots = np.einsum("ij,ij->i", n, grad)
    if euler is None:  # min() of the two distances has no gradient on the plane between the spheres: skip one voxel of it
        dots = dots[np.abs((cen - [0.013, 0.011, 0.021]) @ np.array([1.0, 1.0, 0.0]) / np.sqrt(2)) > vol.voxel_length]
    assert np.all(dots > 0), "a triangle normal points inwards"
    assert np.all(np.abs(sdf(*vd.T)) <= vol.voxel_length / 2)


def test_random_fields_have_no_cracks_between_valid_cubes():
    rng = np.random.default_rng(3)
    res = 20
    vol = T.Volume(2.0, res, 0.1, T.NO_COLOR)
    vol.tw[:, 0] = rng.uniform(-1, 1, res ** 3).astype(np.float32)
    vol.tw[:, 1] = (rng.random(res ** 3) > 0.04).astype(np.float32)
    v, _, t = M.extract_triangle_mesh(vol)
    ci, valid = _cube_indices(vol)
    emit = valid & (ci > 0) & (ci < 255)
    assert len(t) > 3000
    # the cube of every triangle: cubes in index order, mc_tri_count each
    count = np.array([len(G.triangles(k)) for k in range(256)])
    cubes = np.argwhere(emit)
    tri_cube = np.repeat(np.arange(len(cubes)), count[ci[emit]])
    # the grid edge of every vertex, from the definition: crossed and in a valid cube, (x, y, z, axis) order
    f = vol.tw[:, 0].reshape(res, res, res)
    edges = []
    for x in range(res):
        for y in range(res):
            for z in range(res):
                for a in range(3):
                    k = [x, y, z]
                    k[a] += 1
                    if k[a] >= res or (f[x, y, z] < 0) == (f[tuple(k)] < 0):
                        continue
                    c0 = []
                    for d in range(4):
                        c = [x, y, z]
                        c[(a + 1) % 3] -= d & 1
                        c[(a + 2) % 3] -= d >> 1
                        if all(0 <= q <= res - 2 for q in c) and valid[tuple(c)]:
                            c0.append(c)
                    if c0:
                        edges.append((x, y, z, a))
    assert len(edges) == len(v)
    d = _directed_edges(t)
    keys = {}
    for i, (a, b) in enumerate(d):
        assert (int(a), int(b)) not in keys
        keys[(int(a), int(b))] = i % len(t)
    for (a, b), tri in keys.items():
        if (b, a) in keys:
            continue
        # a segment used once lies on a face of its cube whose neighbour across it is not a valid cube
        ea, eb = np.array(edges[a]), np.array(edges[b])
        c = cubes[tri_cube[tri]]
        ok = False
        for ax in range(3):
            if ea[3] == ax or eb[3] == ax or ea[ax] != eb[ax]:
                continue
            nb = c.copy()
            nb[ax] += 1 if ea[ax] == c[ax] + 1 else -1
            ok |= not (all(0 <= q <= res - 2 for q in nb) and valid[tuple(nb)])
        assert ok, "a crack between two valid cubes"


# ------------------------------------------------------------------------------------------------ arithmetic
@pytest.mark.parametrize("ct", [T.NO_COLOR, T.RGB8, T.GRAY32])
def test_vertices_and_colours_against_a_float64_restatement(ct):
    vol = _field_volume(_torus(0.5, 0.22), res=36, ct=ct, seed=7)
    vol.origin[:] = (0.3, -0.2, 0.1)
    v, c, t = M.extract_triangle_mesh(vol)
    if ct == T.NO_COLOR:
        assert c is None
    r, vl = vol.res, float(vol.voxel_length)
    f = vol.tw[:, 0].reshape(r, r, r).astype(np.float64)
    rows, cols = [], []
    ci, valid = _cube_indices(vol)
    for x, y, z in np.argwhere(np.ones((r, r, r), bool)):
        for a in range(3):
            k = [x, y, z]
            k[a] += 1
            if k[a] >= r or (f[x, y, z] < 0) == (f[tuple(k)] < 0):
                continue
            cs = []
            for d in range(4):
                cc = [x, y, z]
                cc[(a + 1) % 3] -= d & 1
                cc[(a + 2) % 3] -= d >> 1
                cs.append(all(0 <= q <= r - 2 for q in cc) and valid[tuple(cc)])
            if not any(cs):
                continue
            f0, f1 = abs(f[x, y, z]), abs(f[tuple(k)])
            p = vl * np.array([x, y, z], np.float64) + vl / 2
            p[a] += f0 * vl / (f0 + f1)
            rows.append(p + vol.origin.astype(np.float64) - (r // 2) * vl)
            if ct != T.NO_COLOR:
                i0, i1 = (x * r + y) * r + z, (k[0] * r + k[1]) * r + k[2]
                pl = vol.col.astype(np.float64) / (255.0 if ct == T.RGB8 else 1.0)
                ch = pl[:, [i0, i1]] if ct == T.RGB8 else np.repeat(pl[:, [i0, i1]], 3, 0)
                cols.append((f1 * ch[:, 0] + f0 * ch[:, 1]) / (f0 + f1))
    ref = np.array(rows)
    assert len(ref) == len(v)
    # a handful of float32 roundings of values up to the grid's extent
    assert np.max(np.abs(v - ref)) <= 8 * np.finfo(np.float32).eps * vol.length
    if ct != T.NO_COLOR:
        rc = np.array(cols)
        assert np.max(np.abs(c - rc) / np.maximum(np.abs(rc), 1e-30)) <= 8 * np.finfo(np.float32).eps


def test_vertex_normals_add_in_ascending_triangle_order():
    rng = np.random.default_rng(11)
    tn = rng.normal(size=(40, 3)).astype(np.float32) * np.float32([1, 1e4, 1e-4])
    # vertex 0 is in every triangle, in varying corners; vertex 1..39 in some
    tris = np.array([np.roll([0, 1 + i % 39, 1 + (i * 7) % 39], i % 3) for i in range(40)], np.int32)
    got = M.vertex_normals(40, tris, tn, normalized=False)
    for v in range(40):
        acc = None
        for c in range(3 * len(tris)):
            if tris.reshape(-1)[c] == v:
                x = tn[c // 3]
                acc = x.copy() if acc is None else (acc + x).astype(np.float32)
        assert np.array_equal(got[v].view(np.uint32), (acc if acc is not None else np.zeros(3, np.float32)).view(np.uint32))
    # (1 + 1e8) - 1e8 is 0 in float32, 1 in any order that adds the large terms first
    tn3 = np.float32([[0, 1, 0], [0, 1e8, 0], [0, -1e8, 0]])
    assert M.vertex_normals(3, np.int32([[0, 1, 2], [1, 0, 2], [2, 1, 0]]), tn3, normalized=False)[0, 1] == 0


def test_unreferenced_vertex_gets_a_zero_normal_and_rows_stay_aligned():
    v = np.float32([[0, 0, 0], [1, 0, 0], [5, 5, 5], [0, 1, 0], [0, 0, 1]])
    t = np.int32([[0, 1, 3], [0, 3, 4], [0, 4, 1]])
    vn, tn = M.compute_vertex_normals(v, t)
    assert vn.shape == (5, 3) and np.all(vn[2] == 0)
    assert np.allclose(vn[1], [0, np.sqrt(0.5), np.sqrt(0.5)]) and np.allclose(vn[3], [np.sqrt(0.5), 0, np.sqrt(0.5)])
    assert np.allclose(tn, [[0, 0, 1], [1, 0, 0], [0, 1, 0]])
    with pytest.raises(ValueError):
        M.triangle_normals(v, np.int32([[0, 1, 5]]))
    with pytest.raises(ValueError):
        M.vertex_normals(5, np.int32([[0, -1, 2]]), tn[:1])


def test_a_vertex_count_past_the_limit_is_refused():
    vol = _field_volume(_sphere((0, 0, 0), 0.6), res=24)
    v, _, _ = M.extract_triangle_mesh(vol)
    assert len(M.extract_triangle_mesh(vol, max_vertices=len(v))[0]) == len(v)
    with pytest.raises(ValueError):
        M.extract_triangle_mesh(vol, max_vertices=len(v) - 1)
