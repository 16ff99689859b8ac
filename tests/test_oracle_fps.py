"""CPU: the FarthestPointDownSample restatement in the oracle against independent numpy restatements.

- Integer lattices (coordinates in [-20, 20], with duplicates): every float32 squared distance is exact, so the oracle
  must equal an int64 farthest-point loop with np.argmax (first maximum) step for step.  These clouds are full of ties
  and pin the tie rule (smallest index among equal distances).
- Random and surface clouds: along the oracle's own pick history, float64 distances to the picks so far; each pick is
  within 1e-6 relative of the float64 maximum, and is the float64 argmax wherever that maximum is clear.
- The quirks of pointcloud.cu:301-338: sample counts 0, 1, n and n + 5, one and no points, identical points, a NaN
  point (it keeps +inf, so once picked it is picked at every later step) and an infinite coordinate."""
import numpy as np
import pytest

from cupoch_b200.testing import datagen


@pytest.fixture(scope="module")
def fpso():
    """the FarthestPointDownSample restatement (oracle/fps.c)"""
    from oracle import fps_py
    fps_py.build()
    return fps_py


def int64_fps(P, k):
    P = np.asarray(P, np.int64)
    dist = np.full(len(P), np.iinfo(np.int64).max, np.int64)
    far, idx = 0, []
    for _ in range(k):
        idx.append(far)
        dist = np.minimum(dist, ((P - P[far]) ** 2).sum(1))
        far = int(np.argmax(dist))
    return np.array(idx, np.int32), dist


def lattice(n, seed, dup_every=7):
    rng = np.random.default_rng(seed)
    P = rng.integers(-20, 21, size=(n, 3))
    P[::dup_every] = P[rng.integers(0, n, size=len(P[::dup_every]))]  # exact duplicates
    return P


@pytest.mark.parametrize("n,k,seed", [(50, 55, 1), (500, 500, 2), (3000, 400, 3), (20000, 300, 4)])
def test_lattice_equals_int64_loop(fpso, n, k, seed):
    P = lattice(n, seed)
    idx, dist = fpso.farthest_point_down_sample(P.astype(np.float32), k)
    ref_idx, ref_dist = int64_fps(P, k)
    np.testing.assert_array_equal(idx, ref_idx)
    np.testing.assert_array_equal(dist.astype(np.int64), ref_dist)


def test_small_lattice_is_all_ties(fpso):
    """a 3x3x3 grid: after the corners every step is a tie; once all 27 points are in, the picks go to index 0"""
    g = np.stack(np.meshgrid(*[np.arange(3)] * 3, indexing="ij"), -1).reshape(-1, 3)
    idx, _ = fpso.farthest_point_down_sample(g.astype(np.float32), 30)
    np.testing.assert_array_equal(idx, int64_fps(g, 30)[0])
    assert sorted(idx[:27].tolist()) == list(range(27)) and idx[27:].tolist() == [0, 0, 0]


def float64_history_check(P, idx):
    """pick t must be (near) the float64 farthest point from picks 0..t-1"""
    P64 = P.astype(np.float64)
    d = np.full(len(P), np.inf)
    clear = 0
    for t in range(1, len(idx)):
        d = np.minimum(d, ((P64 - P64[idx[t - 1]]) ** 2).sum(1))
        top = np.partition(d, len(d) - 2)[-2:]
        mx, second = top[1], top[0]
        assert d[idx[t]] >= mx * (1 - 1e-6), (t, d[idx[t]], mx)
        if second < mx * (1 - 1e-5):
            assert idx[t] == int(np.argmax(d)), t
            clear += 1
    return clear


@pytest.mark.parametrize("kind", ["uniform", "surface"])
def test_float64_history(fpso, kind):
    if kind == "uniform":
        P, k = datagen.uniform_cube(4000, 5, lo=(-1, -2, 0), hi=(3, 2, 1)), 300
    else:
        P, k = datagen.surface(6000, 6)[0], 400
    idx, dist = fpso.farthest_point_down_sample(P, k)
    assert len(set(idx.tolist())) == k  # distinct points: no repeats before n
    clear = float64_history_check(P, idx)
    assert clear > 0.9 * (k - 1)
    # the final distances are the float32 distances to the nearest pick
    d64 = np.min(((P[:, None, :].astype(np.float64) - P[idx][None].astype(np.float64)) ** 2).sum(-1), 1)
    np.testing.assert_allclose(dist, d64, rtol=1e-5, atol=1e-12)


def test_sample_counts(fpso):
    P = datagen.uniform_cube(200, 8)
    n = len(P)
    assert len(fpso.farthest_point_down_sample(P, 0)[0]) == 0
    assert fpso.farthest_point_down_sample(P, 1)[0].tolist() == [0]
    full, dist = fpso.farthest_point_down_sample(P, n)
    assert sorted(full.tolist()) == list(range(n)) and not dist.any()
    more, _ = fpso.farthest_point_down_sample(P, n + 5)
    np.testing.assert_array_equal(more[:n], full)
    assert more[n:].tolist() == [0] * 5  # every distance is 0: the smallest index wins
    # the first picks do not depend on how many are asked for
    np.testing.assert_array_equal(fpso.farthest_point_down_sample(P, 17)[0], full[:17])


def test_one_and_no_points(fpso):
    idx, dist = fpso.farthest_point_down_sample(np.zeros((0, 3), np.float32), 3)
    assert len(idx) == 0 and len(dist) == 0
    idx, dist = fpso.farthest_point_down_sample(np.array([[1, 2, 3]], np.float32), 4)
    assert idx.tolist() == [0, 0, 0, 0] and dist.tolist() == [0.0]


def test_identical_points(fpso):
    idx, dist = fpso.farthest_point_down_sample(np.full((40, 3), 0.25, np.float32), 6)
    assert idx.tolist() == [0] * 6 and not dist.any()


@pytest.mark.parametrize("bad", [[np.nan, 0, 0], [0, np.inf, 0]])
def test_non_finite_point_repeats(fpso, bad):
    """d2 to a NaN point is NaN and fminf ignores it; d2 from an infinite point to itself is inf - inf = NaN: either
    point keeps +inf, wins every later argmax, and no other distance changes after it is picked"""
    P = datagen.uniform_cube(100, 9)
    P[37] = bad
    idx, dist = fpso.farthest_point_down_sample(P, 8)
    assert idx.tolist() == [0] + [37] * 7
    assert np.isinf(dist[37])
    d0 = ((P.astype(np.float64) - P[0]) ** 2).sum(1)
    mask = np.arange(100) != 37
    np.testing.assert_allclose(dist[mask], d0[mask], rtol=1e-6)
