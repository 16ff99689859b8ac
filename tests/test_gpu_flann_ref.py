"""GPU parity against the REFERENCE'S OWN search engine: the FLANN CUDA kd-tree cupoch vendors
(third_party/flann/algorithms/kdtree_cuda_3d_index.cu), called exactly like cupoch::knn::KDTreeFlann calls it
(kdtree_flann.inl:70-144).  Its answers are stored in tests/golden/flann_ref.npz (tools/make_flann_golden.py runs
oracle/_ref/libflann_ref.so, built by oracle/ref_flann/Makefile, on every query of each case below and keeps a fixed,
seeded sample of the rows).  The product searches every query; the sampled rows are compared.  This pins the search
row (SURVEY 8a R1/R1b) to reference CODE, not to a restatement:

  * which point is returned (index) and its d2 -- BIT-IDENTICAL: the product computes d2 in the operation order the
    reference's kernel has in SASS (FMUL dy,dy; FFMA dx,dx; FFMA dz,dz) -- on random clouds and on the ICP workload;
  * the tie rule (DESIGN.md hazard 1): FLANN keeps the first-visited of equal-distance points in kd order, the
    product keeps the smallest index -- measured here, asserted only through d2 (the distances must agree);
  * k > 1 radius results that are not full (R1b, result_set.h:405-473): same SET of neighbours.
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cupoch_b200 as cph
from cupoch_b200.testing import datagen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "flann_ref.npz")


class Flann:
    """FLANN's stored answers for one case: rows = the sampled query indices"""
    def __init__(self, case):
        with np.load(GOLDEN) as g:
            self.rows, self.idx, self.d2 = g[case + "_rows"], g[case + "_idx"], g[case + "_d2"]


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _compare_1nn(case, tgt, qry, r):
    ref = Flann(case)
    tree = cph.geometry.KDTreeFlann(cph.geometry.PointCloud(tgt))
    _, idx, d2 = tree.search_radius(qry, r, 1)
    qry = qry[ref.rows]
    idx, d2 = idx.cpu()[ref.rows, 0], d2.cpu()[ref.rows, 0]
    fi, fd = ref.idx[:, 0], ref.d2[:, 0]
    found, ffound = idx >= 0, fi >= 0
    both = found & ffound
    # a query whose nearest point lies within an ulp of the radius may be in on one side and out on the other
    # (FLANN's d2 is compiled with --use_fast_math contraction, ours follows the written contract)
    edge = found != ffound
    u = _ulps(d2[both], fd[both])
    idx_diff = both & (idx != fi)
    # where the indices differ the two points must be (numerically) equidistant: a tie, not a wrong answer
    tie_ok = True
    if idx_diff.any():
        q = qry[idx_diff].astype(np.float64)
        da = ((q - tgt[idx[idx_diff]].astype(np.float64)) ** 2).sum(1)
        db = ((q - tgt[fi[idx_diff]].astype(np.float64)) ** 2).sum(1)
        tie_ok = bool(np.all(np.abs(da - db) <= 4e-7 * np.maximum(da, db) + 1e-30))
    assert tie_ok, "product and FLANN return different, non-equidistant points"
    assert edge.sum() <= max(2, len(qry) // 100000)
    if edge.any():  # those must sit on the radius
        de = np.where(found[edge], d2[edge], fd[edge])
        assert np.all(np.abs(de - np.float32(r) * np.float32(r)) <= 4e-7 * de)
    # d2 follows the operation order the reference's kernel has in SASS (cphb_internal.cuh dist2): bit-identical
    assert (u == 0).all(), "d2 differs from the reference binary's in %d of %d results" % (int((u != 0).sum()), len(u))
    return int(idx_diff.sum())


def test_flann_1nn_uniform():
    tgt = datagen.uniform_cube(200_000, 101)
    qry = datagen.uniform_cube(100_000, 202, lo=(-0.05, -0.05, -0.05), hi=(1.05, 1.05, 1.05))
    assert _compare_1nn("uniform_r0.02", tgt, qry, 0.02) <= 5          # random floats: ties are essentially impossible
    _compare_1nn("uniform_r0.3", tgt, qry, 0.3)


def test_flann_1nn_icp_workload():
    # the first search of config 2 (misaligned surface), 1 M -> 1 M
    tgt, _ = datagen.surface(1_000_000, 11)
    src = datagen.make_source(tgt, datagen.gt_transform(), 13, 14, 5e-4)
    assert _compare_1nn("config2", tgt, src, 0.02) <= 20


def test_flann_ties():
    # lattice + duplicates, queries at cell centres / on lattice points: every query has several equidistant
    # nearest points.  d2 must agree bit for bit (all values are exact in float); the INDEX is the tie rule.
    g = np.stack(np.meshgrid(*[np.arange(12, dtype=np.float32)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.25
    tgt = np.concatenate([g, g[::3], g[::7]]).astype(np.float32)
    tgt = tgt[np.random.default_rng(3).permutation(len(tgt))]
    qry = np.concatenate([g + 0.125, g]).astype(np.float32)
    ref = Flann("lattice")
    assert np.array_equal(ref.rows, np.arange(len(qry)))
    fi, fd = ref.idx, ref.d2
    tree = cph.geometry.KDTreeFlann(cph.geometry.PointCloud(tgt))
    _, idx, d2 = tree.search_radius(qry, 0.5, 1)
    idx, d2 = idx.cpu(), d2.cpu()
    np.testing.assert_array_equal(d2, fd)
    # both answers are nearest points; ours is the smallest index among them
    d_ours = ((qry - tgt[idx[:, 0]]) ** 2).sum(1)
    d_ref = ((qry - tgt[fi[:, 0]]) ** 2).sum(1)
    np.testing.assert_array_equal(d_ours, d_ref)
    assert (idx[:, 0] <= fi[:, 0]).all()


@pytest.mark.parametrize("k,r", [(4, 0.05), (15, 0.08), (30, 0.1)])
def test_flann_radius_k_not_full(k, r):
    # R1b: radius search with max_nn > 1 where most result lists are NOT full.  The reference heap-sorts an array it
    # only heapifies on the k-th insert (result_set.h:405-473): compare as sets
    tgt = datagen.uniform_cube(20_000, 5)
    qry = datagen.uniform_cube(5_000, 6)
    ref = Flann("radius_k%d" % k)
    fi = ref.idx
    tree = cph.geometry.KDTreeFlann(cph.geometry.PointCloud(tgt))
    _, idx, d2 = tree.search_radius(qry, r, k)
    idx = idx.cpu()[ref.rows]
    same_set = np.array([set(a[a >= 0].tolist()) == set(b[b >= 0].tolist()) for a, b in zip(idx, fi)])
    n_found = (idx >= 0).sum(1)
    full = n_found == k
    # lists that are not full contain EVERY point inside the radius on both sides: the sets must be equal.  A full
    # list may differ only where the k-th and (k+1)-th neighbour tie.
    assert same_set[~full].all()
    assert same_set.mean() > 0.999


def test_flann_knn30():
    tgt = datagen.uniform_cube(50_000, 7)
    qry = datagen.uniform_cube(5_000, 8)
    ref = Flann("knn30")
    fi, fd = ref.idx, ref.d2
    tree = cph.geometry.KDTreeFlann(cph.geometry.PointCloud(tgt))
    _, idx, d2 = tree.search_knn(qry, 30)
    idx, d2 = idx.cpu()[ref.rows], d2.cpu()[ref.rows]
    same_set = np.array([set(a.tolist()) == set(b.tolist()) for a, b in zip(idx, fi)])
    assert same_set.mean() > 0.999
    assert _ulps(np.sort(d2, 1), np.sort(fd, 1)).max() == 0
