"""CPU: the ComputeSHOTFeature oracle (oracle/shot.c) checked three ways.

- Against the independent float64 restatement cupoch_b200.testing.shot64 on the oracle's own neighbour lists: points
  whose computation stays clear of every decision (margin > SLACK) match to ATOL per bin; the others are counted and
  must stay a small fraction.
- Invariants: every row has unit norm or is all zero; a rigid motion of cloud and normals leaves the rows of points away
  from the decisions unchanged within tolerance.
- One test per behaviour the reference has and the library keeps, and per deliberate deviation (DESIGN.md hazard 14).
The quirk clouds are shared with tests/test_gpu_shot.py."""
import numpy as np
import pytest

from cupoch_b200.testing import datagen, shot64

SPACING = 1.0 / np.sqrt(1e5)  # datagen.surface at 1e5 points per unit square
R = float(np.float32(5 * SPACING))
SLACK = 1e-4                  # decision margin (relative) below which float32 may take the other branch
ATOL = 5e-5                   # per-bin agreement of the points above it
MAX_UNSTABLE = 0.30           # fraction of points allowed within SLACK of a decision


@pytest.fixture(scope="module")
def shoto():
    from oracle import shot_py
    shot_py.build()
    return shot_py


def cloud(n, seed):
    return datagen.surface(n, seed, extent=float(np.sqrt(n / 1e5)))


def planar_lattice(side):
    """side x side unit lattice on z = 0 with +z normals: frame coordinates land exactly on sector boundaries"""
    g = np.arange(side, dtype=np.float32)
    x, y = np.meshgrid(g, g, indexing="ij")
    pts = np.stack([x.ravel(), y.ravel(), np.zeros(side * side, np.float32)], 1).astype(np.float32)
    return pts, np.tile(np.float32([0, 0, 1]), (len(pts), 1))


def star():
    """a point with its 6 axis neighbours at distance exactly 1: with radius 1 every frame weight is 0, w_total == 0"""
    pts = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    return pts, np.tile(np.float32([0.6, 0.0, 0.8]), (7, 1))


def few(m, dup=False):
    """m points on a small circle around the origin (plus the origin, and a duplicate of it when dup)"""
    a = np.linspace(0, 2 * np.pi, m, endpoint=False)
    ring = np.stack([np.cos(a), np.sin(a), 0.1 * np.sin(3 * a)], 1) * 0.3
    pts = np.concatenate([[[0, 0, 0]], ring] + ([[[0, 0, 0]]] if dup else [])).astype(np.float32)
    return pts, np.tile(np.float32([0, 0, 1]), (len(pts), 1))


def quirk_clouds():
    """name -> (points, normals, radius, (knn, search_radius, max_nn))"""
    pts, nrm = cloud(3000, 21)
    dup = np.concatenate([pts, pts[:300]]), np.concatenate([nrm, nrm[:300]])
    lat = planar_lattice(12)
    return {
        "surface_radius": (pts, nrm, R, (0, R, 100)),
        "neighbour_normals_randomised": (pts, _randomise_others(nrm), R, (0, R, 100)),
        "own_normal_flipped": (pts, -nrm, R, (0, R, 100)),
        "duplicates": (dup[0], dup[1], R, (0, R, 100)),
        "knn_beyond_radius": (pts, nrm, 0.5 * R, (30, 0.0, 0)),
        "search_wider": (pts, nrm, R, (0, 2.0 * R, 256)),
        "four_neighbours": (*few(4), 1.0, (0, 1.0, 100)),
        "five_neighbours": (*few(5), 1.0, (0, 1.0, 100)),
        "four_and_duplicate": (*few(4, True), 1.0, (0, 1.0, 100)),
        "w_total_zero": (*star(), 1.0, (7, 0.0, 0)),
        "step10_lattice": (lat[0], lat[1], 2.5, (0, 2.5, 100)),
        "step0_lattice": (lat[0], -lat[1], 2.5, (0, 2.5, 100)),
        "tiny_search": (pts, nrm, R, (0, 0.0, 100)),
    }


def _randomise_others(nrm):
    """odd rows get random unit normals, even rows keep theirs"""
    rng = np.random.default_rng(3)
    out = nrm.copy()
    r = rng.normal(size=(len(nrm[1::2]), 3))
    out[1::2] = (r / np.linalg.norm(r, axis=1, keepdims=True)).astype(np.float32)
    return out


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("search", [(0, R, 100), (0, 1.6 * R, 256), (30, 0.0, 0), (100, 0.0, 0), (10, 0.0, 0)])
def test_matches_float64_restatement(shoto, search):
    pts, nrm = cloud(2500, 5)
    radius = R if search != (10, 0.0, 0) else 0.5 * R  # kNN lists reaching past the descriptor radius
    idx, d2 = shoto.neighbours(pts, *search)
    f = shoto.compute_shot_feature(pts, nrm, radius, *search)
    np.testing.assert_array_equal(bits(f), bits(shoto.shot_from_neighbours(pts, nrm, idx, d2, radius)))
    g, margin = shot64.shot64(pts, nrm, idx, d2, radius)
    stable = margin > SLACK
    assert (~stable).mean() <= MAX_UNSTABLE, (~stable).mean()
    err = np.abs(f - g).max(1)
    assert err[stable].max() <= ATOL, err[stable].max()
    assert (np.abs(f).sum(1) > 0).mean() > 0.9


@pytest.mark.parametrize("search", [(0, R, 100), (30, 0.0, 0), (0, 2.0 * R, 256)])
def test_unit_norm_or_zero(shoto, search):
    pts, nrm = cloud(5000, 9)
    f = shoto.compute_shot_feature(pts, nrm, R, *search).astype(np.float64)
    norms = np.linalg.norm(f, axis=1)
    zero = ~f.any(1)
    assert np.all(np.isfinite(f))
    assert np.all(zero | (np.abs(norms - 1) < 1e-5))
    assert (~zero).mean() > 0.9


def test_rigid_motion_invariance(shoto):
    pts, nrm = cloud(3000, 13)
    c, s = np.cos(0.7), np.sin(0.7)
    Rm = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]) @ np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    t = np.array([0.3, -0.2, 0.1])
    pts2 = (pts.astype(np.float64) @ Rm.T + t).astype(np.float32)
    nrm2 = (nrm.astype(np.float64) @ Rm.T).astype(np.float32)
    search = (0, R, 100)
    f1 = shoto.compute_shot_feature(pts, nrm, R, *search)
    f2 = shoto.compute_shot_feature(pts2, nrm2, R, *search)
    idx1, d21 = shoto.neighbours(pts, *search)
    idx2, d22 = shoto.neighbours(pts2, *search)
    m1 = shot64.shot64(pts, nrm, idx1, d21, R)[1]
    m2 = shot64.shot64(pts2, nrm2, idx2, d22, R)[1]
    same_lists = np.array([set(a[a >= 0]) == set(b[b >= 0]) for a, b in zip(idx1, idx2)])
    stable = (m1 > SLACK) & (m2 > SLACK) & same_lists
    assert stable.mean() > 0.3
    assert np.abs(f1 - f2)[stable].max() < 1e-3


def test_own_normal_quirk(shoto):
    """cos_desc uses the point's own normal for every neighbour (shot.cu:115): other points' normals never matter, all
    of a row's mass sits in one or two cosine columns, and flipping the point's normal mirrors the columns"""
    pts, nrm = cloud(3000, 21)
    f = shoto.compute_shot_feature(pts, nrm, R, 0, R, 100)
    g = shoto.compute_shot_feature(pts, _randomise_others(nrm), R, 0, R, 100)
    np.testing.assert_array_equal(bits(f[0::2]), bits(g[0::2]))
    assert np.any(bits(f[1::2]) != bits(g[1::2]))
    cols = (f.reshape(-1, 32, 11) != 0).any(1)
    assert np.all(cols.sum(1)[f.any(1)] <= 2)
    h = shoto.compute_shot_feature(pts, -nrm, R, 0, R, 100).reshape(-1, 32, 11)
    # columns c <-> 10 - c, except where the cosine interpolation wraps ((step + 1) % 10 at step 9)
    mirrored = np.all((h != 0).any(1)[:, ::-1] == cols, axis=1) & f.any(1)
    assert mirrored.mean() > 0.9
    np.testing.assert_allclose(h[mirrored][:, :, ::-1], f.reshape(-1, 32, 11)[mirrored], atol=1e-5)


def test_step_index_10_column(shoto):
    """cos_desc = 1 gives step_index 10 (:142): the 11th column of a volume, hence 32 x 11 = 352 bins"""
    pts, nrm = planar_lattice(12)
    up = shoto.compute_shot_feature(pts, nrm, 2.5, 0, 2.5, 100).reshape(-1, 32, 11)
    down = shoto.compute_shot_feature(pts, -nrm, 2.5, 0, 2.5, 100).reshape(-1, 32, 11)
    col = lambda f, c: np.abs(f[:, :, c]).sum(1) > 0  # noqa: E731
    # the frame's z is +-e_z exactly, so one orientation of the normal gives cos_desc = 1, the other -1
    hit10 = col(up, 10) | col(down, 10)
    assert hit10.mean() > 0.5
    for f in (up, down):
        assert np.all(np.isfinite(f)) and np.all(np.abs(f).sum((1, 2)) > 0)
        c10 = col(f, 10)
        assert np.all(np.abs(f[c10][:, :, 1:9]).sum((1, 2)) == 0)  # cos_desc ~ 1: columns 9 / 10 only


def test_duplicates(shoto):
    """self is skipped by index only: a coincident duplicate enters the frame with w = radius (and counts towards the
    5) but adds nothing to the histogram (dist == 0, :114)"""
    p4, n4 = few(4)
    p4d, n4d = few(4, True)
    assert not shoto.compute_shot_feature(p4, n4, 1.0, 0, 1.0, 100)[0].any()  # 4 frame neighbours: zero row
    f = shoto.compute_shot_feature(p4d, n4d, 1.0, 0, 1.0, 100)
    assert f[0].any() and f[-1].any()  # 4 + the duplicate: 5 frame neighbours
    pts, nrm = cloud(3000, 21)
    dp, dn = np.concatenate([pts, pts[:300]]), np.concatenate([nrm, nrm[:300]])
    fd = shoto.compute_shot_feature(dp, dn, R, 0, R, 100)
    assert np.any(bits(fd[:300]) != bits(shoto.compute_shot_feature(pts, nrm, R, 0, R, 100)[:300]))


def test_fewer_than_five_neighbours_zero_row(shoto):
    for m, nonzero in ((4, False), (5, True)):
        pts, nrm = few(m)
        f = shoto.compute_shot_feature(pts, nrm, 1.0, 0, 1.0, 100)
        assert f[0].any() == nonzero
        assert not f[1:].any() or m == 5  # each ring point sees the centre and its ring: m others
    pts, nrm = cloud(2000, 4)
    assert not shoto.compute_shot_feature(pts, nrm, R, 5, 0.0, 0).any()  # KNN 5 = self + 4
    assert not shoto.compute_shot_feature(pts, nrm, R, 0, R, 0).any()    # max_nn = 0
    assert not shoto.compute_shot_feature(pts, nrm, R, 0, 0.0, 100).any()  # search radius 0 lists nothing


def test_knn_beyond_radius(shoto):
    """radius is independent of the search: neighbours past it get negative frame weights and shell weights outside
    [0, 1]; the float64 restatement follows them"""
    pts, nrm = cloud(2500, 8)
    idx, d2 = shoto.neighbours(pts, 30)
    assert (np.sqrt(d2[:, -1]) > 0.5 * R).mean() > 0.9
    f = shoto.compute_shot_feature(pts, nrm, 0.5 * R, 30)
    g, margin = shot64.shot64(pts, nrm, idx, d2, 0.5 * R)
    stable = margin > SLACK
    assert stable.mean() > 1 - MAX_UNSTABLE
    assert np.abs(f - g)[stable].max() <= ATOL
    assert np.any(bits(f) != bits(shoto.compute_shot_feature(pts, nrm, R, 30)))


def test_w_total_zero_degenerate_frame(shoto):
    """every frame weight 0: NaN covariance, FastEigen3x3's identity branch, min id == max id -> x = z, y = 0; the row
    is kept (finite, unit norm)"""
    pts, nrm = star()
    f = shoto.compute_shot_feature(pts, nrm, 1.0, 7)
    assert np.all(np.isfinite(f[0])) and abs(np.linalg.norm(f[0].astype(np.float64)) - 1) < 1e-5


def test_empty_single_and_illegal(shoto):
    assert shoto.compute_shot_feature(np.zeros((0, 3)), np.zeros((0, 3)), R, 30).shape == (0, 352)
    one = shoto.compute_shot_feature(np.zeros((1, 3)), np.float32([[0, 0, 1]]), R, 30)
    assert one.shape == (1, 352) and not one.any()
    pts, nrm = cloud(100, 1)
    for bad in ((101, 0.0, 0), (0, R, 257), (0, R, -1)):
        with pytest.raises(ValueError):
            shoto.compute_shot_feature(pts, nrm, R, *bad)
    shoto.compute_shot_feature(pts, nrm, R, 100)
    shoto.compute_shot_feature(pts, nrm, R, 0, R, 256)
