"""CPU: the mesh voxelisation restatement (oracle/mesh_voxel.c).  Its cell-major loop (the reference's enumeration) and
its triangle-major enumeration agree on random meshes, on vertices lying exactly on cell faces, edges and corners, on
segments, points, triangles larger than the grid or partly outside it, and on non-finite vertices; the centre rule's
known answers; every decision of the float32 test that differs from a float64 restatement lies within rounding of the
separating threshold; points sampled on a mesh away from cell faces fall in voxels; the count rule and every rejection."""
import numpy as np
import pytest

from oracle import mesh_voxel_py as MV

LO, HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)


def both(v, t, vs, lo=LO, hi=HI):
    a = MV.voxelize(v, t, vs, lo, hi, MV.CELL_MAJOR)
    b = MV.voxelize(v, t, vs, lo, hi, MV.TRIANGLE_MAJOR)
    assert np.array_equal(a, b), (len(a), len(b))
    return a


@pytest.mark.parametrize("seed", range(6))
def test_cell_major_equals_triangle_major_on_random_meshes(seed):
    rng = np.random.default_rng(seed)
    v = (rng.normal(size=(40, 3)) * 0.6).astype(np.float32)
    t = rng.integers(0, 40, (30, 3)).astype(np.int32)
    assert len(both(v, t, float(rng.choice([0.1, 0.125, 0.2, 0.3])))) > 0


@pytest.mark.parametrize("seed", range(4))
def test_vertices_on_cell_faces_edges_and_corners(seed):
    rng = np.random.default_rng(10 + seed)
    v = (rng.integers(-12, 13, (30, 3)) / 8.0).astype(np.float32)  # dyadic: every coordinate on a face of vs = 1/8 cells
    t = rng.integers(0, 30, (40, 3)).astype(np.int32)
    both(v, t, 0.125)
    both(v + np.float32(1 / 16), t, 0.125)  # on the cell centres' planes


def test_segments_points_big_and_partly_outside_triangles():
    v = np.array([[0.0, 0.0, 0.0], [1.0, 0.5, 0.25], [-9.0, -9.0, 0.1], [9.0, -9.0, 0.1], [0.0, 9.0, 0.1], [1.4, 1.4, 1.4],
                  [2.5, 1.0, 1.0], [0.25, 0.25, 0.25]], np.float32)
    seg, pt, big, out, corner = [0, 0, 1], [7, 7, 7], [2, 3, 4], [5, 6, 0], [1, 1, 1]
    k = both(v, [seg], 0.25)
    assert len(k) >= 5
    k = both(v, [pt], 0.25)  # a point on a corner shared by 8 cells
    assert len(k) == 8
    assert len(both(v, [corner], 0.25)) >= 1
    assert len(both(v, [big], 0.25)) == 12 * 12  # the plane z = 0.1 through the whole grid, one layer
    assert len(both(v, [out], 0.25)) > 0


def test_non_finite_vertices_meet_no_cell():
    rng = np.random.default_rng(3)
    v = (rng.normal(size=(20, 3)) * 0.5).astype(np.float32)
    t = rng.integers(3, 20, (15, 3)).astype(np.int32)
    want = both(v, t, 0.125)
    v[0], v[1], v[2] = (np.nan, 0, 0), (np.inf, 0.1, 0), (0, -np.inf, 0)
    t2 = np.concatenate([t, [[0, 3, 4], [1, 5, 6], [2, 7, 8], [0, 1, 2]]]).astype(np.int32)
    assert np.array_equal(both(v, t2, 0.125), want)


def test_the_centre_rule_known_answers():
    """a triangle in the plane z = o_z + 0.75 vs: cell k_z = 0 with the true centre, k_z = 1 with the reference's
    lower-corner centre"""
    v = np.array([[0.1, 0.1, 0.375], [1.9, 0.1, 0.375], [0.1, 1.9, 0.375]], np.float32)
    for mode in (MV.CELL_MAJOR, MV.TRIANGLE_MAJOR):
        k = MV.voxelize(v, [[0, 1, 2]], 0.5, (0, 0, 0), (2, 2, 2), mode)
        c = MV.voxelize(v, [[0, 1, 2]], 0.5, (0, 0, 0), (2, 2, 2), mode, corner=True)
        assert set(k[:, 2]) == {0} and set(c[:, 2]) == {1}
        assert len(k) == 13 and len(c) == 14  # the cells (x, y) the triangle reaches under each rule


def sat64(centre, h, tri):
    """the separating-axis test in float64 -> (overlap, margin): the margin is the smallest slack over the 13 axes in
    distance units when they overlap, minus the largest separation when they do not"""
    v = np.asarray(tri, np.float64) - np.asarray(centre, np.float64)
    e = [v[1] - v[0], v[2] - v[1], v[0] - v[2]]
    axes = [np.eye(3)[a] for a in range(3)] + [np.cross(np.eye(3)[a], ed) for ed in e for a in range(3)]
    axes.append(np.cross(e[0], e[1]))
    slack, sep = np.inf, -np.inf
    for a in axes:
        n = np.linalg.norm(a)
        if n == 0:
            continue
        p = v @ a
        r = h * np.abs(a).sum()
        s = min(r - p.min(), p.max() + r) / n
        slack, sep = min(slack, s), max(sep, -s)
    return (sep <= 0), (slack if sep <= 0 else -sep)


@pytest.mark.parametrize("seed", range(3))
def test_float32_decisions_against_a_float64_restatement(seed):
    rng = np.random.default_rng(20 + seed)
    vs, h = 0.125, 0.0625
    diffs, n = [], 0
    for _ in range(150):
        tri = (rng.normal(size=(3, 3)) * 0.3).astype(np.float32)
        lo = np.floor(tri.min(0) / vs).astype(int) - 1
        hi = np.floor(tri.max(0) / vs).astype(int) + 1
        for x in range(lo[0], hi[0] + 1):
            for y in range(lo[1], hi[1] + 1):
                for z in range(lo[2], hi[2] + 1):
                    c = ((np.array([x, y, z], np.float32) + np.float32(0.5)) * np.float32(vs)).astype(np.float32)
                    got = MV.tri_box(c, h, *tri)
                    want, margin = sat64(c, h, tri)
                    n += 1
                    if got != want:
                        diffs.append((tuple(tri.ravel()), (x, y, z), got, margin))
    print("%d decisions, %d differ from float64:" % (n, len(diffs)))
    for d in diffs:
        print("  triangle %s cell %s float32 %s margin %.3g" % d)
    assert n > 10000
    assert all(abs(d[3]) <= 1e-6 for d in diffs)


def test_sampled_points_away_from_faces_are_in_their_voxels():
    rng = np.random.default_rng(5)
    v = (rng.normal(size=(60, 3)) * 0.6).astype(np.float32)
    t = rng.integers(0, 60, (80, 3)).astype(np.int32)
    vs, o = np.float32(0.1), np.float32(-1.5)
    keys = {tuple(k) for k in MV.voxelize(v, t, vs, LO, HI)}
    w = rng.dirichlet((1, 1, 1), size=(len(t), 20))
    p = np.einsum("tsj,tjq->tsq", w, v[t].astype(np.float64)).reshape(-1, 3)
    q = (p - o) / vs
    away = (np.abs(q - np.round(q)) > 1e-5).all(1) & (q >= 0).all(1) & (q < 30).all(1)
    assert away.sum() > 1000
    cells = np.floor(q[away]).astype(int)
    assert all(tuple(c) in keys for c in cells)


def test_count_rule_and_rejections():
    assert MV.counts(0.5, (0, 0, 0), (2, 1.2, 1.3)) == (4, 2, 3)  # roundf: 2.4 -> 2, 2.6 -> 3
    assert MV.counts(1.0, (0, 0, 0), (0.5, 1.5, 2.0 ** 21 - 1.5)) == (1, 2, 2 ** 21 - 1)  # halves round away from zero
    v, t = np.zeros((3, 3), np.float32), np.array([[0, 1, 2]], np.int32)
    for vs, lo, hi in ((0.0, LO, HI), (-1.0, LO, HI), (np.nan, LO, HI), (np.inf, LO, HI), (0.1, (np.nan, 0, 0), HI),
                       (0.1, LO, (np.inf, 0, 0)), (0.1, (1, 0, 0), (-1, 1, 1)), (1.0, (0, 0, 0), (2.0 ** 21, 1, 1)),
                       (1.0, (0, 0, 0), (1, 1, 2.0 ** 21 - 0.5))):
        with pytest.raises(ValueError):
            MV.counts(vs, lo, hi)
        with pytest.raises(ValueError):
            MV.voxelize(v, t, vs, lo, hi)
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        with pytest.raises(ValueError):
            MV.voxelize(v, bad, 0.5, LO, HI)
    assert len(MV.voxelize(v, np.zeros((0, 3), np.int32), 0.5, LO, HI)) == 0
    assert len(MV.voxelize(v, t, 0.5, (0, 0, 0), (0, 1, 1))) == 0  # zero cells on an axis
