"""CPU: the ComputeISSKeypoints restatement (oracle/iss.c) pinned three ways.

- Against an independent float64 restatement in numpy on the oracle's own neighbour lists: float64 cumulants and
  covariance, np.linalg.eigvalsh of the covariance divided by its largest coefficient, the ratio tests and the
  suppression.  Saliencies agree to SAL_TOL times the float32 covariance's cancellation error; masks agree except at
  points whose decision lies within that tolerance of a threshold or of a neighbour's saliency, and those are few.
- At the reference's quirks, one test each.
- On a known answer: a lattice on the surface of a box has a keypoint within 2 x resolution of each of its 8 corners."""
import numpy as np
import pytest

from cupoch_b200.testing import datagen

SAL_TOL = 4.0  # |saliency - float64| <= SAL_TOL * kappa, kappa = the float32 covariance's cancellation (saliency64)


@pytest.fixture(scope="module")
def isso():
    from oracle import iss_py
    iss_py.build()
    return iss_py


@pytest.fixture(scope="module")
def orc():
    from oracle import oracle_py
    oracle_py.build()
    return oracle_py


def box_lattice(m, seed=0):
    """the lattice points (i, j, k) / m of [0, 1]^3 with a coordinate on a face, rows shuffled: every 2-NN distance is 1/m"""
    g = np.arange(m + 1)
    P = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    P = P[((P == 0) | (P == m)).any(1)]
    return (P[np.random.default_rng(seed).permutation(len(P))] / np.float32(m)).astype(np.float32)


def saliency64(pts, idx, min_neighbors=5, gamma_21=0.975, gamma_32=0.975):
    """-> (saliency, tolerance, ambiguous, l1) in float64 from neighbour lists idx [n, k] (-1 = empty).  The float32
    covariance E[xx^T] - E[x]E[x]^T cancels: its error is about 2^-23 max|E[xx^T]|, so a normalised eigenvalue is good
    to about kappa = 2^-23 max|E[xx^T]| / (largest covariance coefficient); tolerance = SAL_TOL * kappa."""
    P = pts.astype(np.float64)
    ok = idx >= 0
    cnt = ok.sum(1)
    nb = P[np.where(ok, idx, 0)] * ok[..., None]
    c = np.maximum(cnt, 1)[:, None]
    mean = nb.sum(1) / c
    m2 = np.einsum("nki,nkj->nij", nb, nb) / c[..., None]
    cov = m2 - mean[:, :, None] * mean[:, None, :]
    flat = cov.reshape(len(P), 9)
    mc = flat.max(1)
    off = np.abs(cov[:, [0, 0, 1], [1, 2, 2]]).max(1) > 0
    scale = np.where(off & (mc > 0), mc, 1.0)  # FastEigen3x3 normalises in its general branch only
    ev = np.linalg.eigvalsh(cov / scale[:, None, None])
    l1, l2, l3 = ev[:, 0], ev[:, 1], ev[:, 2]
    tol = SAL_TOL * 2.0 ** -23 * np.abs(m2).reshape(len(P), 9).max(1) / scale
    zero = (np.abs(flat) <= 1e-5).all(1)
    good = (cnt >= min_neighbors) & ~zero & (l3 > 0) & (l2 < gamma_21 * l3) & (l1 < gamma_32 * l2)
    # ambiguous: a ratio test or isZero within tolerance of its threshold, or the sign of l1 (a negative float32 saliency
    # passes the ratio tests and is then suppressed by the saliency >= 0 test)
    amb = (cnt >= min_neighbors) & ((np.abs(l2 - gamma_21 * l3) <= 2 * tol) | (np.abs(l1 - gamma_32 * l2) <= 2 * tol)
                                   | (np.abs(l1) <= tol) | (np.abs(np.abs(flat).max(1) - 1e-5) <= 1e-5 * 2.0 ** -10))
    return np.where(good, l1, -1.0), tol, amb, l1


def nms(sal, idx):
    """is_local_maxima_functor on lists idx [n, k]: saliency >= 0 and no listed neighbour strictly larger"""
    ok = idx >= 0
    nb = np.where(ok, sal[np.where(ok, idx, 0)], -np.inf)
    return (sal >= 0) & ~(nb > sal[:, None]).any(1)


@pytest.mark.parametrize("n,radii", [(4000, (0.0, 0.0)), (4000, (0.08, 0.05)), (20000, (0.06, 0.04))])
def test_float64_restatement(isso, orc, n, radii):
    # centred on the origin: the float32 covariance then cancels least, which keeps the ambiguous decisions few
    pts = datagen.surface(n, 11 + n % 7)[0] - np.float32([0.5, 0.5, 0.0])
    mask, sal, (rs, rn) = isso.iss_keypoints(pts, *radii)
    idx_s = orc.search(pts, pts, 100, float(rs), kdtree=True)[0]
    idx_n = orc.search(pts, pts, 100, float(rn), kdtree=True)[0]
    s64, tol, amb, l1 = saliency64(pts, idx_s)
    both = (sal >= 0) & (s64 >= 0)
    err = np.abs(sal[both] - s64[both]) / tol[both]
    print("n=%d: %d salient, max saliency error / tolerance %.2f, %d ambiguous" % (n, both.sum(), err.max(), amb.sum()))
    assert (err <= 1).all()
    assert both.sum() > n // 10
    flip = (sal >= 0) != (s64 >= 0)
    assert not (flip & ~amb).any()
    # suppression: a decision is certain when a neighbour is surely more salient, or every neighbour surely less; the
    # float32 value of an ambiguous point is -1 or about its l1
    m64 = nms(np.where(amb, sal, s64), idx_n)
    ok = (idx_n >= 0) & (idx_n != np.arange(n)[:, None])
    j = np.where(ok, idx_n, 0)
    hi = np.where(amb, np.maximum(l1, -1.0), s64) + tol
    lo = np.where(amb, -1.0, s64 - tol)
    hi_i, lo_i = hi[:, None], lo[:, None]
    suppressed = (ok & (lo[j] > hi_i)).any(1)
    kept = (s64 >= 0) & ~amb & ~(ok & (hi[j] >= lo_i)).any(1)
    shaky = ~((s64 < 0) & ~amb) & ~suppressed & ~kept
    diff = mask != m64
    print("  %d keypoints, %d near a threshold or tie, %d differ from float64" % (mask.sum(), shaky.sum(), diff.sum()))
    assert not (diff & ~shaky).any()
    assert shaky.sum() <= 0.02 * n and mask.sum() > 0


def test_both_radii_replaced_when_one_is_zero(isso):
    pts = datagen.surface(5000, 3)[0]
    _, _, auto = isso.iss_keypoints(pts)
    for given in ((0.2, 0.0), (0.0, 0.2), (-0.0, 0.3)):
        m, s, r = isso.iss_keypoints(pts, *given)
        np.testing.assert_array_equal(r, auto)
    m, s, r = isso.iss_keypoints(pts, 0.2, 0.1)
    np.testing.assert_array_equal(r, np.float32([0.2, 0.1]))
    assert auto[0] == np.float32(6) * (auto[0] / np.float32(6)) and auto[0] != np.float32(0.2)


def test_resolution_is_root_mean_square(isso):
    """two planar lattices far apart, spacings 1/16 and 1/4: every 2-NN distance is the spacing, so the sum of squares is
    exact and resolution = sqrt((nA a^2 + nB b^2) / n), not the mean distance"""
    a, b = 1 / 16, 1 / 4
    A = np.stack(np.meshgrid(np.arange(20), np.arange(20), [0], indexing="ij"), -1).reshape(-1, 3) * a
    B = np.stack(np.meshgrid(np.arange(6), np.arange(6), [0], indexing="ij"), -1).reshape(-1, 3) * b + 100.0
    pts = np.concatenate([A, B]).astype(np.float32)
    n = len(pts)
    _, _, r = isso.iss_keypoints(pts)
    res = np.sqrt(np.float32((len(A) * a * a + len(B) * b * b)) / np.float32(n))
    assert res.dtype == np.float32
    np.testing.assert_array_equal(r, [np.float32(6) * res, np.float32(4) * res])
    assert abs(res - (len(A) * a + len(B) * b) / n) > 0.01


def test_iszero_is_absolute(isso):
    pts = box_lattice(16)
    m1, _, _ = isso.iss_keypoints(pts)
    m3, s3, r3 = isso.iss_keypoints(pts * np.float32(1e-3))
    assert m1.sum() > 8
    assert m3.sum() == 0 and (s3 == -1).all() and r3[0] > 0


def _cluster(centre, half, R):
    """the centre and +-half[i] along the rotated axes R[:, i]: 7 points, mean = centre"""
    off = [np.zeros(3)] + [s * h * R[:, i] for i, h in enumerate(half) for s in (1, -1)]
    return (np.asarray(centre) + np.array(off)).astype(np.float32)


def test_normalised_saliency_decides_suppression(isso):
    """cluster A is smaller than cluster B in absolute smallest eigenvalue but larger once each covariance is divided by its
    largest coefficient: the normalised values decide, so A's points suppress B's centre"""
    c, s = np.cos(0.6), np.sin(0.6)
    R = np.array([[1, 0, 0], [0, c, -s], [0, s, c]]) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    A = _cluster((0, 0, 0), (0.10, 0.09, 0.08), R)
    B = _cluster((1, 0, 0), (0.20, 0.16, 0.13), R)
    pts = np.concatenate([A, B])
    absl, norm = [], []
    for X in (A, B):
        cov = np.cov(X.astype(np.float64).T, bias=True)
        ev = np.linalg.eigvalsh(cov)
        absl.append(ev[0])
        norm.append(ev[0] / cov.max())
    assert absl[0] < absl[1] and norm[0] > norm[1]  # the premise
    # min_neighbors = 7: only the points that see their whole cluster within 0.25 are salient (all of A, B's centre)
    mask, sal, _ = isso.iss_keypoints(pts, 0.25, 1.5, min_neighbors=7)
    assert (sal[:7] >= 0).all() and sal[7] >= 0 and (sal[8:] == -1).all()
    assert len(set(sal[:7].tolist())) == 1  # identical neighbourhoods, identical saliency
    assert mask[:7].all() and not mask[7:].any()


def test_strict_comparison_keeps_equal_neighbours(isso):
    P = box_lattice(16)
    pts = np.concatenate([P, P])  # every point has an exact duplicate with the same neighbourhood
    mask, sal, _ = isso.iss_keypoints(pts, 0.375, 0.25, max_neighbors=256)
    n = len(P)
    np.testing.assert_array_equal(sal[:n], sal[n:])
    np.testing.assert_array_equal(mask[:n], mask[n:])
    assert mask.sum() >= 16


def test_min_neighbors_boundary(isso, orc):
    pts = datagen.surface(3000, 5)[0]
    r = 0.04
    cnt = (orc.search(pts, pts, 100, r, kdtree=True)[0] >= 0).sum(1)
    _, s_all, _ = isso.iss_keypoints(pts, r, r, min_neighbors=0)
    c = int(np.median(cnt))
    for mn in (c - 1, c, c + 1):
        _, s, _ = isso.iss_keypoints(pts, r, r, min_neighbors=mn)
        np.testing.assert_array_equal(s[cnt < mn], -1)
        np.testing.assert_array_equal(s[cnt >= mn], s_all[cnt >= mn])
    assert ((cnt == c) & (s_all >= 0)).any()


def test_max_neighbors_truncates_suppression_window(isso, orc):
    pts = datagen.surface(4000, 6)[0]
    rs, rn = 0.05, 0.05
    masks = {}
    for k in (8, 100):
        mask, sal, _ = isso.iss_keypoints(pts, rs, rn, max_neighbors=k)
        idx = orc.search(pts, pts, k, rn, kdtree=True)[0]
        np.testing.assert_array_equal(mask, nms(sal.astype(np.float64), idx))
        masks[k] = mask
    # the same saliencies with the full window: truncation keeps points a farther, more salient one would suppress
    _, sal8, _ = isso.iss_keypoints(pts, rs, rn, max_neighbors=8)
    full = nms(sal8.astype(np.float64), orc.search(pts, pts, 100, rn, kdtree=True)[0])
    assert (masks[8] & ~full).any() and not (full & ~masks[8]).any()


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_fewer_than_five_points_give_nothing(isso, n):
    pts = datagen.uniform_cube(n, 1)
    mask, sal, r = isso.iss_keypoints(pts)
    assert not mask.any() and (sal == -1).all()
    if n == 1:
        assert np.isinf(r).all()


def test_coincident_points_give_nothing(isso):
    pts = np.full((500, 3), 0.25, np.float32)
    mask, sal, r = isso.iss_keypoints(pts)
    np.testing.assert_array_equal(r, [0, 0])
    assert not mask.any() and (sal == -1).all()


def test_empty_and_illegal(isso):
    m, s, r = isso.iss_keypoints(np.zeros((0, 3), np.float32), 0.1, 0.2)
    assert len(m) == 0 and len(s) == 0
    np.testing.assert_array_equal(r, np.float32([0.1, 0.2]))
    with pytest.raises(ValueError):
        isso.iss_keypoints(datagen.uniform_cube(10, 1), max_neighbors=257)
    m, s, _ = isso.iss_keypoints(datagen.uniform_cube(100, 1), 0.5, 0.5, min_neighbors=0, max_neighbors=0)
    assert not m.any() and (s == -1).all()


@pytest.mark.parametrize("m", [16, 32, 64])
def test_box_corners_known_answer(isso, m):
    pts = box_lattice(m, seed=m)
    mask, _, r = isso.iss_keypoints(pts)
    res = r[0] / np.float32(6)
    assert res == np.float32(1 / m)  # every 2-NN distance is 1/m: the root mean square is exact
    corners = np.array([[i, j, k] for i in (0, 1) for j in (0, 1) for k in (0, 1)], np.float32)
    d = np.linalg.norm(pts[mask][None] - corners[:, None], axis=2).min(1)
    assert (d <= 2 * res).all(), d / res
