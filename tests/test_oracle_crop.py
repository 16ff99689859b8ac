"""CPU: the bounding-box selection and cleanup restatement (oracle/crop.c) -- pinned to the reference's known answers
(tests/golden/pointcloud_crop_known.json, from tools/make_golden.py), to plain numpy for the three predicates, and to a
float64 PCA for the oriented box."""
import json
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cp():
    from oracle import crop_py
    crop_py.build()
    return crop_py


@pytest.fixture(scope="module")
def known():
    with open(os.path.join(ROOT, "tests", "golden", "pointcloud_crop_known.json")) as f:
        return json.load(f)


def _sorted_rows(a):
    a = np.asarray(a, np.float64)
    return a[np.lexsort(a.T[::-1])]


# ---- the reference's known answers -----------------------------------------------------------------------------------
def test_golden_oriented_bounding_box(cp, known):
    g = known["oriented_bounding_box"]
    c, R, e = cp.obb_create(g["points_8"])
    np.testing.assert_array_equal(c, np.float32(g["center"]))
    np.testing.assert_array_equal(e, np.float32(g["extent"]))
    np.testing.assert_array_equal(R, np.float32(g["R"]))
    np.testing.assert_array_equal(_sorted_rows(cp.obb_box_points(c, R, e)), _sorted_rows(g["box_points"]))
    c4, R4, e4 = cp.obb_create(g["points_4"])  # the reference only asks that this runs
    assert np.isfinite(c4).all() and np.isfinite(R4).all() and np.isfinite(e4).all()


def test_golden_normalize_normals(cp, known):
    g = known["normalize_normals"]
    np.testing.assert_allclose(cp.normalize_normals(g["normals"]), g["ref"], atol=known["tolerance"])


def test_golden_uniform_down_sample(cp, known):
    g = known["uniform_down_sample"]
    pts = np.float32(g["points"])
    rows = cp.uniform_rows(len(pts), g["every_k_points"])
    np.testing.assert_allclose(pts[rows], g["ref"], atol=known["tolerance"])


def test_golden_crop(cp, known):
    g = known["crop"]
    pts = np.float32(g["points"])
    kept = cp.aabb_indices(pts, g["min_bound"], g["max_bound"])
    assert 0 < len(kept) < len(pts)
    assert (pts[kept] >= np.float32(g["min_bound"])).all() and (pts[kept] <= np.float32(g["max_bound"])).all()
    dropped = np.setdiff1d(np.arange(len(pts)), kept)
    assert ((pts[dropped] < 200) | (pts[dropped] > 800)).any(axis=1).all()


def test_golden_orient_normals(cp, known):
    from oracle import oracle_py as orc
    g = known["orient_normals"]
    nrm = orc.estimate_normals(np.float32(g["points"]), knn=g["knn"])
    np.testing.assert_allclose(cp.orient_normals(nrm, g["reference"]), g["ref"], atol=known["tolerance"])


# ---- predicates against plain numpy ---------------------------------------------------------------------------------
def _edge_cloud(seed, n=4000):
    """random points on a coarse lattice (many exactly on the bounds) with NaN, +-inf and -0.0 coordinates mixed in"""
    rng = np.random.default_rng(seed)
    pts = (rng.integers(-4, 5, (n, 3)) * 0.25).astype(np.float32)
    specials = np.float32([np.nan, np.inf, -np.inf, -0.0, 0.0])
    mask = rng.random((n, 3)) < 0.08
    pts[mask] = rng.choice(specials, mask.sum())
    return pts


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_aabb_matches_numpy(cp, seed):
    pts = _edge_cloud(seed)
    lo, hi = np.float32([-0.5, -0.0, -1.0]), np.float32([0.5, 0.75, 0.0])
    drop = ((pts < lo) | (pts > hi)).any(axis=1)
    np.testing.assert_array_equal(cp.aabb_indices(pts, lo, hi), np.flatnonzero(~drop))
    assert np.isnan(pts[cp.aabb_indices(pts, lo, hi)]).any()  # NaN points are kept


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_pass_through_matches_numpy(cp, axis):
    pts = _edge_cloud(10 + axis)
    v = pts[:, axis]
    keep = ~((v < np.float32(-0.25)) | (np.float32(0.5) < v))
    np.testing.assert_array_equal(cp.pass_through_indices(pts, axis, -0.25, 0.5), np.flatnonzero(keep))


@pytest.mark.parametrize("rm_nan,rm_inf", [(True, True), (True, False), (False, True), (False, False)])
def test_finite_matches_numpy(cp, rm_nan, rm_inf):
    pts = _edge_cloud(20)
    drop = np.zeros(len(pts), bool)
    if rm_nan:
        drop |= np.isnan(pts).any(axis=1)
    if rm_inf:
        drop |= np.isinf(pts).any(axis=1)
    np.testing.assert_array_equal(cp.finite_indices(pts, rm_nan, rm_inf), np.flatnonzero(~drop))


def _rotation(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_obb_containment_matches_signed_distance(cp, seed):
    rng = np.random.default_rng(100 + seed)
    R = _rotation(seed).astype(np.float32)
    c = rng.uniform(-5, 5, 3).astype(np.float32)
    e = rng.uniform(0.5, 3, 3).astype(np.float32)
    box = cp.obb_box_points(c, R, e)
    pts = (c + rng.uniform(-1, 1, (20000, 3)) * e.max()).astype(np.float32)
    # float64 signed distance to every face, in the box frame
    local = (pts.astype(np.float64) - c.astype(np.float64)) @ R.astype(np.float64)
    margin = np.abs(local) - e.astype(np.float64) / 2  # > 0 outside along that axis
    inside = (margin < 0).all(axis=1)
    clear = np.abs(margin).min(axis=1) > 1e-4  # farther than this from every face plane
    got = np.zeros(len(pts), bool)
    got[cp.obb_indices(pts, box)] = True
    assert clear.sum() > 0.95 * len(pts)
    np.testing.assert_array_equal(got[clear], inside[clear])


def test_obb_degenerate_box_is_whatever_the_determinants_give(cp):
    """a zero extent makes some plane triples collinear (determinant 0 for every point), so the test no longer describes
    the flat box: (2, 0, 0) outside it is kept and (0.25, 0.25, 0.1) just above it is dropped.  Pinned as the
    reference's determinants give it."""
    box = cp.obb_box_points([0, 0, 0], np.eye(3), [1, 1, 0])
    pts = np.float32([[0, 0, 0], [0.25, 0.25, 0], [0.25, 0.25, 0.1], [2, 0, 0], [0.5, 0.5, 0]])
    np.testing.assert_array_equal(cp.obb_indices(pts, box), [0, 1, 3, 4])


# ---- OBB creation against a float64 PCA -----------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4])
def test_obb_create_matches_float64_pca(cp, seed):
    rng = np.random.default_rng(200 + seed)
    R0 = _rotation(seed)
    half = np.array([3.0, 1.5, 0.5]) * rng.uniform(0.5, 2)
    pts = ((rng.uniform(-1, 1, (5000, 3)) * half) @ R0.T + rng.uniform(-10, 10, 3)).astype(np.float32)
    c, R, e = cp.obb_create(pts)
    p = pts.astype(np.float64)
    mean = p.mean(0)
    w, V = np.linalg.eigh(np.cov((p - mean).T, bias=True))
    V = V[:, ::-1]  # descending eigenvalues
    for k in range(3):
        assert abs(abs(np.dot(R[:, k].astype(np.float64), V[:, k])) - 1) < 1e-5
    local = (p - mean) @ V
    e64 = local.max(0) - local.min(0)
    c64 = V @ ((local.max(0) + local.min(0)) / 2) + mean
    np.testing.assert_allclose(e, e64, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(c, c64, atol=1e-3)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_obb_invariants(cp, seed):
    rng = np.random.default_rng(300 + seed)
    pts = (rng.normal(size=(3000, 3)) * rng.uniform(0.1, 5, 3) + rng.uniform(-50, 50, 3)).astype(np.float32)
    c, R, e = cp.obb_create(pts)
    R64 = R.astype(np.float64)
    np.testing.assert_allclose(R64.T @ R64, np.eye(3), atol=1e-6)
    for k in range(3):  # the sign rule: each axis' largest-magnitude component is positive
        assert R[np.argmax(np.abs(R[:, k])), k] > 0
    local = (pts.astype(np.float64) - c) @ R64
    assert (np.abs(local) <= e / 2 + 1e-3).all()


def test_obb_empty_and_single(cp):
    c, R, e = cp.obb_create(np.zeros((0, 3), np.float32))
    np.testing.assert_array_equal(R, np.eye(3, dtype=np.float32))
    assert not c.any() and not e.any()
    c, R, e = cp.obb_create(np.float32([[1, 2, 3]]))
    np.testing.assert_array_equal(c, [1, 2, 3])
    np.testing.assert_array_equal(R, np.eye(3, dtype=np.float32))
    assert not e.any()


# ---- uniform stride and normals ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,k", [(0, 1), (1, 1), (10, 3), (12, 4), (5, 7), (100, 1)])
def test_uniform_rows(cp, n, k):
    np.testing.assert_array_equal(cp.uniform_rows(n, k), np.arange(n // k) * k)


def test_uniform_rejects_zero(cp):
    assert cp.uniform_rows(10, 0) is None


def test_normal_operations_edge_cases(cp):
    nrm = np.float32([[0, 0, 0], [3, 4, 0], [-1, 0, 0], [0, 0, -0.0], [1e-30, 0, 0], [np.nan, 0, 0], [0, -2, 0]])
    out = cp.normalize_normals(nrm)
    np.testing.assert_array_equal(out[[0, 3]], nrm[[0, 3]])  # zero stays zero
    np.testing.assert_array_equal(out[1], np.float32([0.6, 0.8, 0]))
    np.testing.assert_array_equal(out[4], nrm[4])  # |n|^2 underflows to 0: unchanged, as Eigen's normalize()
    assert np.isnan(out[5, 0])
    o = cp.orient_normals(nrm, [1, 0, 0])
    np.testing.assert_array_equal(o[0], [1, 0, 0])           # zero -> the reference
    np.testing.assert_array_equal(o[2], [1, 0, 0])           # pointing away -> negated
    np.testing.assert_array_equal(o[6], nrm[6])              # orthogonal: dot == 0 is not < 0
    np.testing.assert_array_equal(o[5, 1:], nrm[5, 1:])      # NaN compares false: unchanged
