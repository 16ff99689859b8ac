"""CPU: oracle/mesh_clean.c -- hand-worked answers for the four Remove* operations and operator+='s triangles, the
TriangleTriangle3d predicate on hand-built pairs, the all-pairs loop (with the finite / box filter) against the
sort-and-sweep mode, the unfiltered loop agreeing with the filtered one away from degenerate input, a nearly degenerate
pair the reference reports with disjoint boxes, and every rejection."""
import numpy as np
import pytest

from oracle import mesh_clean_py as MC


def test_remove_duplicated_vertices_by_hand():
    v = np.array([[1, 0, 0], [0, 0, 0], [1, 0, 0], [-0.0, 0, 0], [np.nan, 0, 0], [0, 1, 0], [np.nan, 0, 0]], np.float32)
    n = np.arange(21, dtype=np.float32).reshape(7, 3)
    t = np.array([[0, 1, 5], [2, 3, 6], [4, 5, 0]], np.int32)
    ov, ot, on, _ = MC.remove_duplicated_vertices(v, t, normals=n)
    # sorted distinct positions: (0,0,0) from 1 (and -0 from 3), (0,1,0) from 5, (1,0,0) from 0 (and 2); NaNs 4, 6 last
    assert np.array_equal(ov[:3], np.array([[0, 0, 0], [0, 1, 0], [1, 0, 0]], np.float32))
    assert np.isnan(ov[3, 0]) and np.isnan(ov[4, 0]) and len(ov) == 5
    assert np.array_equal(on, n[[1, 5, 0, 4, 6]])
    assert np.array_equal(ot, [[2, 0, 1], [2, 0, 4], [3, 1, 2]])


def test_remove_duplicated_triangles_by_hand():
    t = np.array([[2, 0, 1], [0, 1, 2], [1, 2, 0], [0, 2, 1], [3, 1, 2], [0, 1, 2]], np.int32)
    tn = np.arange(18, dtype=np.float32).reshape(6, 3)
    ot, otn = MC.remove_duplicated_triangles(t, 4, tn)
    assert np.array_equal(ot, [[0, 1, 2], [0, 2, 1], [1, 2, 3]])
    assert np.array_equal(otn, tn[[0, 3, 4]])


def test_remove_unreferenced_and_degenerate_by_hand():
    v = np.arange(15, dtype=np.float32).reshape(5, 3)
    t = np.array([[4, 1, 1], [1, 4, 3]], np.int32)
    ov, ot, _, oc = MC.remove_unreferenced_vertices(v, t, colors=v * 2)
    assert np.array_equal(ov, v[[1, 3, 4]]) and np.array_equal(oc, v[[1, 3, 4]] * 2)
    assert np.array_equal(ot, [[2, 0, 0], [0, 2, 1]])
    ot, otn = MC.remove_degenerate_triangles(t, 5, None)
    assert np.array_equal(ot, [[1, 4, 3]]) and otn is None
    assert np.array_equal(MC.append_triangles(t, 5, [[0, 1, 2]], 3), [[4, 1, 1], [1, 4, 3], [5, 6, 7]])


def test_every_rejection():
    v = np.zeros((3, 3), np.float32)
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        with pytest.raises(ValueError):
            MC.remove_duplicated_vertices(v, bad)
        with pytest.raises(ValueError):
            MC.remove_unreferenced_vertices(v, bad)
        with pytest.raises(ValueError):
            MC.remove_duplicated_triangles(bad, 3)
        with pytest.raises(ValueError):
            MC.remove_degenerate_triangles(bad, 3)
        with pytest.raises(ValueError):
            MC.self_intersections(v, bad)
        with pytest.raises(ValueError):
            MC.append_triangles([[0, 1, 2]], 3, bad, 3)


def test_predicate_by_hand():
    p = [[0, 0, 0], [1, 0, 0], [0, 1, 0]]
    assert MC.tritri(p, [[0.2, 0.2, -1], [0.2, 0.2, 1], [0.3, 0.25, 1]])        # piercing
    assert not MC.tritri(p, [[0.2, 0.2, 0.1], [0.6, 0.2, 1], [0.3, 0.5, 1]])    # above
    assert MC.tritri(p, [[0.1, 0.1, 0], [0.9, 0.05, 0], [0.2, 0.6, 0]])         # coplanar overlapping
    assert not MC.tritri(p, [[2, 2, 0], [3, 2, 0], [2, 3, 0]])                  # coplanar disjoint
    assert not MC.tritri(p, [[0, 0, 1], [1, 0, 1], [0, 1, 1]])                  # parallel planes


def soup(seed, n, scale=1.0, size=0.2, shift=10.0):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-scale, scale, (n, 1, 3))
    v = (c + rng.normal(size=(n, 3, 3)) * size).reshape(-1, 3).astype(np.float32)
    v = (v + np.float32(shift)).astype(np.float32)  # away from the origin, so the normalisation is exercised
    return v, np.arange(3 * n, dtype=np.int32).reshape(n, 3)


def coplanar_grid(k=12):
    xs = np.arange(k, dtype=np.float32) * 0.5
    v, t = [], []
    for x in xs:
        for y in xs:
            b = len(v)
            v += [[x, y, 0], [x + 0.7, y, 0], [x, y + 0.7, 0]]
            t.append([b, b + 1, b + 2])
    return np.array(v, np.float32), np.array(t, np.int32)


def shared_positions(seed):
    """a welded mesh's positions under different indices: every vertex appears twice"""
    rng = np.random.default_rng(seed)
    base = rng.uniform(0, 1, (60, 3)).astype(np.float32)
    v = np.concatenate([base, base])
    t = rng.integers(0, 120, (200, 3)).astype(np.int32)
    return v, t


def degenerate(seed):
    rng = np.random.default_rng(seed)
    v, t = soup(seed, 150, 0.5, 0.3)
    t[::7, 1] = t[::7, 0]                       # segments by index
    v[t[::5, 2]] = v[t[::5, 0]]                 # segments by position
    v[t[::11, 1]] = v[t[::11, 0]] + np.float32(1e-6) * rng.normal(size=(len(t[::11]), 3)).astype(np.float32)
    return v, t


@pytest.mark.parametrize("case", ["soup", "coplanar", "shared", "degenerate"])
def test_all_pairs_filtered_equals_sweep(case):
    v, t = {"soup": lambda: soup(1, 300, 1.0, 0.3), "coplanar": coplanar_grid, "shared": lambda: shared_positions(2),
            "degenerate": lambda: degenerate(3)}[case]()
    a = MC.self_intersections(v, t, MC.ALL_PAIRS, True)
    b = MC.self_intersections(v, t, MC.SWEEP)
    assert np.array_equal(a, b)
    assert len(a) > 0


@pytest.mark.parametrize("seed", [4, 5, 6])
def test_filter_matters_only_on_degenerate_input(seed):
    v, t = soup(seed, 250, 1.0, 0.3)
    assert np.array_equal(MC.self_intersections(v, t, MC.ALL_PAIRS, False), MC.self_intersections(v, t, MC.ALL_PAIRS, True))


def test_a_nearly_degenerate_pair_with_disjoint_boxes():
    # a sliver (first triangle) whose normal puts every |du| below the epsilon goes down the coplanar branch, which
    # tests a 2-D projection only: the reference reports it against a triangle whose box it does not meet in z
    p = np.array([[0.2872645854949951, 0.37904199957847595, 0.07535285502672195],
                  [0.23967215418815613, 2.0061774253845215, -2.1800949573516846],
                  [0.28256720304489136, 0.5396468639373779, -0.1472688615322113]], np.float32)
    q = np.array([[0.007020788732916117, 0.23991015553474426, 0.2607246935367584],
                  [0.5759153962135315, 0.7755484580993652, 0.274660587310791],
                  [0.7661830186843872, 0.8215019106864929, 0.6571909785270691]], np.float32)
    assert MC.tritri(p, q)
    v = np.concatenate([p, q])
    t = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    assert np.array_equal(MC.self_intersections(v, t, MC.ALL_PAIRS, False), [[0, 1]])
    assert len(MC.self_intersections(v, t, MC.ALL_PAIRS, True)) == 0


def test_non_finite_vertices_are_dropped_by_the_filter():
    v, t = soup(7, 40, 0.3, 0.3)
    v[0] = (np.inf, 0, 0)
    v[5] = (np.nan, 0, 0)
    f = MC.self_intersections(v, t, MC.ALL_PAIRS, True)
    assert not np.isin(f, [0, 1]).any()
    assert np.array_equal(f, MC.self_intersections(v, t, MC.SWEEP))


def _golden():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tritri_ref.npz"))
    return g["p"], g["q"], g["hit"], g["kind"]


def test_predicate_equals_the_reference_header_on_every_golden_pair():
    # tests/golden/tritri_ref.npz holds the answers of the reference's own opttritri.h (tools/make_tritri_golden.py)
    p, q, hit, kind = _golden()
    got = np.array([MC.tritri(a, b) for a, b in zip(p, q)], np.uint8)
    bad = np.nonzero(got != hit)[0]
    assert len(bad) == 0, (bad[:10], kind[bad[:10]])
    for k in range(9):  # every family is present, and the epsilon family decides both ways
        assert (kind == k).sum() > 0
    assert 0 < hit[kind == 6].sum() < (kind == 6).sum()
