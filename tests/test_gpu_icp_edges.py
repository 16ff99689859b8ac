"""GPU parity of the fused ICP loop (icp_kernels.cuh, icp.cu) where a nearest-neighbour search usually breaks: exact
ties and duplicate targets, degenerate clouds, targets and sources past 1 048 576 points, and the loop's stop rules.

Exact steps: on a 1/4-spaced lattice with dyadic offsets, axis normals and signed-permutation poses every coordinate,
distance, Jacobian entry and product is exact, so any float64 summation order gives the same bits.  The kernel's
correspondences and sums must then equal a plain numpy brute force (smallest d2, then smallest index) and numpy
float64 sums, with no tolerance.  Everything else is compared with the CPU oracle: pose within 1e-5 Frobenius,
identical iterations and correspondence sets, fitness and rmse within 1e-6."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cupoch_b200 as cph
from cupoch_b200.testing import datagen, features64

R = cph.registration
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POSE_TOL = 1e-5  # Frobenius, BASELINE.json north_star
EXACT_R = 0.5    # r2 = 0.25 exactly; every lattice query's nearest site is within 3/64


def cloud(p, n=None, c=None, cov=None):
    pc = cph.geometry.PointCloud(p)
    if n is not None:
        pc.normals = n
    if c is not None:
        pc.colors = c
    if cov is not None:
        pc.covariances = cov
    return pc


def _compare(res, ref):
    d = np.linalg.norm(res.transformation.astype(np.float64) - ref["transformation"].astype(np.float64))
    assert d <= POSE_TOL, "pose differs by %g (Frobenius)" % d
    assert res.iterations == ref["iterations"]
    assert abs(res.fitness - ref["fitness"]) <= 1e-6
    assert abs(res.inlier_rmse - ref["inlier_rmse"]) <= 1e-6
    np.testing.assert_array_equal(res.correspondence_set, ref["correspondence_set"])


def _same_bits(a, b):
    np.testing.assert_array_equal(a.transformation, b.transformation)
    np.testing.assert_array_equal(a.correspondence_set, b.correspondence_set)
    assert a.iterations == b.iterations and a.fitness == b.fitness and a.inlier_rmse == b.inlier_rmse


def sums_to_f32_equal(a, b, idx):
    """both sides are float64 sums of identical float32 products in different orders: equal after float32 rounding
    except on a rounding boundary (<= 1 ulp)"""
    a32, b32 = a[idx].astype(np.float32), b[idx].astype(np.float32)
    np.testing.assert_allclose(a[idx], b[idx], rtol=1e-10, atol=1e-12 * np.abs(a[idx]).max())
    assert (np.abs(a32.view(np.int32) - b32.view(np.int32)) <= 1).all()


# ---- exact inputs ---------------------------------------------------------------------------------------------------
def _axis_vectors(rng, n):
    v = np.zeros((n, 3), np.float32)
    v[np.arange(n), rng.integers(0, 3, n)] = rng.choice(np.array([-1.0, 1.0], np.float32), n)
    return v


def exact_target(m, seed):
    """m sites of the 1/4-spaced lattice, one in eight a copy of another (with its normal), rows shuffled; normals
    +-e_i"""
    rng = np.random.Generator(np.random.PCG64(seed))
    n_dup = m // 8
    n_uni = m - n_dup
    side = 1
    while side ** 3 < n_uni:
        side += 1
    sites = rng.choice(side ** 3, n_uni, replace=False)
    g = np.stack(np.unravel_index(sites, (side,) * 3), 1).astype(np.float32) * np.float32(0.25)
    nrm = _axis_vectors(rng, n_uni)
    pick = rng.integers(0, n_uni, n_dup)
    p, n = np.concatenate([g, g[pick]]), np.concatenate([nrm, nrm[pick]])
    perm = rng.permutation(m)
    return np.ascontiguousarray(p[perm]), np.ascontiguousarray(n[perm])


def exact_queries(n, tgt, seed):
    """target sites plus: nothing (d2 = 0, ties among duplicates), an edge midpoint (2 equidistant sites), a face
    centre (4), a cell centre (8), an offset with one nearest site, or a step far out of range"""
    rng = np.random.Generator(np.random.PCG64(seed))
    base = tgt[rng.integers(0, len(tgt), n)].astype(np.float64)
    e = 0.125
    kinds = rng.integers(0, 6, n)
    off = np.zeros((n, 3))
    for i, k in enumerate(kinds):
        if k == 1:
            off[i, rng.integers(0, 3)] = e
        elif k == 2:
            off[i, rng.choice(3, 2, replace=False)] = e
        elif k == 3:
            off[i] = e
        elif k == 4:
            off[i] = rng.permutation([1 / 32, 1 / 16, 3 / 64])
        elif k == 5 and rng.random() < 0.3:
            off[i, 2] = 64.0
    off *= rng.choice([-1.0, 1.0], (n, 3))
    return (base + off).astype(np.float32)


def signed_permutation(perm, signs, t):
    T = np.zeros((4, 4), np.float32)
    T[np.arange(3), perm] = signs
    T[:3, 3] = t
    T[3, 3] = 1
    return T


POSES = [np.eye(4, dtype=np.float32),
         signed_permutation([1, 2, 0], [-1, 1, -1], [0.5, -1.25, 2.0]),
         signed_permutation([2, 0, 1], [1, -1, 1], [-0.75, 0.25, -3.5])]


def pull_back(P, T):
    """source points that T maps exactly onto P"""
    Rm, t = T[:3, :3].astype(np.float64), T[:3, 3].astype(np.float64)
    return ((P.astype(np.float64) - t) @ Rm).astype(np.float32)


def brute_force(P, tgt, r):
    """nearest target of every query by exact float64 d2, the smallest index among equal d2; -1 unless d2 < r^2.
    Queries on the 1/64 grid and targets on the 1/4 grid below 2^7 in magnitude: |q|^2 + |t|^2 - 2 q.t has at most
    ~30 significant bits in every partial sum, so the expanded form (one float64 GEMM) is exact whatever its order."""
    for a, unit in ((P, 64), (tgt, 4)):
        assert np.array_equal(np.round(a.astype(np.float64) * unit), a.astype(np.float64) * unit) and np.abs(a).max() < 128
    T64 = tgt.astype(np.float64)
    tt = (T64 * T64).sum(1)
    r2 = float(np.float32(r) * np.float32(r))
    idx = np.full(len(P), -1, np.int32)
    d2 = np.zeros(len(P))
    for s in range(0, len(P), 1024):
        q = P[s:s + 1024].astype(np.float64)
        D = (q * q).sum(1)[:, None] + tt[None, :] - 2.0 * (q @ T64.T)
        j = D.argmin(1)  # first minimum = smallest index
        dj = D[np.arange(len(q)), j]
        ok = dj < r2
        idx[s:s + 1024] = np.where(ok, j, -1)
        d2[s:s + 1024] = dj
    return idx, d2


def _jtj_sums(J, r):
    S = np.zeros(32)
    p = 0
    for a in range(6):
        for b in range(a, 6):
            S[p] = (J[:, a] * J[:, b]).sum()
            p += 1
    S[21:27] = (J * r[:, None]).sum(0)
    S[27] = (r * r).sum()
    return S


def p2plane_sums64(P, tgt, tn, ci, d2):
    m = ci >= 0
    s, t, n = P[m].astype(np.float64), tgt[ci[m]].astype(np.float64), tn[ci[m]].astype(np.float64)
    S = _jtj_sums(np.concatenate([np.cross(s, n), n], 1), ((s - t) * n).sum(1))
    S[28], S[29] = d2[m].sum(), m.sum()
    return S


def symmetric_sums64(P, sn, tgt, tn, ci, d2):
    m = ci >= 0
    s, t = P[m].astype(np.float64), tgt[ci[m]].astype(np.float64)
    nn = sn[m].astype(np.float64) + tn[ci[m]]
    S = _jtj_sums(np.concatenate([np.cross(s + t, nn), nn], 1), ((s - t) * nn).sum(1))
    S[28], S[29] = d2[m].sum(), m.sum()
    return S


def p2p_sums64(P, tgt, ci, d2):
    """orc_kabsch_sums layout: sum s, sum t, sum s_a t_b; d2 sum in 28, count in 29"""
    m = ci >= 0
    s, t = P[m].astype(np.float64), tgt[ci[m]].astype(np.float64)
    S = np.zeros(32)
    S[0:3], S[3:6] = s.sum(0), t.sum(0)
    S[6:15] = (s[:, :, None] * t[:, None, :]).sum(0).reshape(9)
    S[28], S[29] = d2[m].sum(), m.sum()
    return S


SRC_COUNTS = [1, 31, 33, 1000, 7936, 8193]      # 7936 / 8193: either side of the 64-block grid (certified helpers)
TGT_COUNTS = [1, 32, 33, 1024, 1025, 32768, 32769]  # index depth 0 -> 1 -> 2


@pytest.mark.parametrize("m", TGT_COUNTS)
@pytest.mark.parametrize("n", SRC_COUNTS)
def test_exact_step_p2plane_p2p(orc, n, m):
    """one search plus sums (IcpContext.step) on exact inputs: indices and sums equal the numpy references bit for bit"""
    tgt, tn = exact_target(m, 100 + m)
    P0 = exact_queries(n, tgt, 200 + n)
    src = pull_back(P0, POSES[1])
    ctx_pl = R.IcpContext(cloud(src), cloud(tgt, tn), EXACT_R, R.TransformationEstimationPointToPlane())
    ctx_pp = R.IcpContext(cloud(src), cloud(tgt), EXACT_R, R.TransformationEstimationPointToPoint())
    try:
        for T in POSES:
            P = orc.transform_points(src, T)
            if T is POSES[1]:
                np.testing.assert_array_equal(P, P0)
            ci_ref, d2 = brute_force(P, tgt, EXACT_R)
            sums, ci = ctx_pl.step(T)
            np.testing.assert_array_equal(ci, ci_ref)
            np.testing.assert_array_equal(sums[:30], p2plane_sums64(P, tgt, tn, ci_ref, d2)[:30])
            sums, ci = ctx_pp.step(T)
            np.testing.assert_array_equal(ci, ci_ref)
            ref = p2p_sums64(P, tgt, ci_ref, d2)
            live = np.r_[0:15, 28, 29]
            np.testing.assert_array_equal(sums[live], ref[live])
    finally:
        ctx_pl.close()
        ctx_pp.close()


def test_exact_queries_tie():
    """the inputs above do what they claim: most matched queries sit on an exact tie between two or more targets"""
    tgt, _ = exact_target(32768, 100 + 32768)
    P = exact_queries(8193, tgt, 200 + 8193)
    ci, d2 = brute_force(P, tgt, EXACT_R)
    T64 = tgt.astype(np.float64)
    m = ci >= 0
    ties = np.array([(((T64 - q) ** 2).sum(1) == d).sum() for q, d in zip(P[m].astype(np.float64), d2[m])])
    assert (ties >= 2).mean() > 0.5 and (ties >= 8).any() and (ties == 1).any() and (~m).any()


@pytest.mark.parametrize("n,m", [(1000, 1025), (8193, 32769)])
def test_exact_step_symmetric(orc, n, m):
    """symmetric rows (s + t) x (n_s + n_t) stay exact too: device = numpy = oracle, bit for bit"""
    tgt, tn = exact_target(m, 300 + m)
    rng = np.random.Generator(np.random.PCG64(n))
    P0 = exact_queries(n, tgt, 400 + n)
    sn0 = _axis_vectors(rng, n)
    T = POSES[2]
    Tr = T.copy()
    Tr[:3, 3] = 0
    src, sn = pull_back(P0, T), pull_back(sn0, Tr)
    ctx = R.IcpContext(cloud(src, sn), cloud(tgt, tn), EXACT_R, R.TransformationEstimationSymmetricMethod())
    try:
        sums, ci = ctx.step(T)
    finally:
        ctx.close()
    P, snm = orc.transform_points(src, T), orc.transform_normals(sn, T)
    np.testing.assert_array_equal(P, P0)
    np.testing.assert_array_equal(snm, sn0)
    ci_ref, d2 = brute_force(P, tgt, EXACT_R)
    np.testing.assert_array_equal(ci, ci_ref)
    ref = symmetric_sums64(P, snm, tgt, tn, ci_ref, d2)
    np.testing.assert_array_equal(sums[:30], ref[:30])
    m_ = ci_ref >= 0
    corr = np.stack([np.nonzero(m_)[0], ci_ref[m_]], 1).astype(np.int32)
    np.testing.assert_array_equal(orc.jtj_jtr(orc.SYMMETRIC, P, tgt, corr, src_nrm=snm, tgt_nrm=tn)[:28], ref[:28])


def _spd(rng, n):
    A = rng.normal(size=(n, 3, 3)) * 0.01
    return (A @ A.transpose(0, 2, 1) + 1e-4 * np.eye(3)).astype(np.float32)


@pytest.mark.parametrize("n,m", [(1000, 1025), (8193, 32769)])
def test_exact_step_colored_gicp(orc, n, m):
    """colored and GICP rows are not exact: the sums agree with the oracle's to 1 ulp after float32 rounding, on
    correspondences that still equal the brute force exactly"""
    tgt, tn = exact_target(m, 500 + m)
    rng = np.random.Generator(np.random.PCG64(m))
    P0 = exact_queries(n, tgt, 600 + n)
    T = POSES[1]
    src = pull_back(P0, T)
    tc, sc = datagen.texture(tgt), rng.random((n, 3), dtype=np.float32)
    P = orc.transform_points(src, T)
    ci_ref, _ = brute_force(P, tgt, EXACT_R)
    m_ = ci_ref >= 0
    corr = np.stack([np.nonzero(m_)[0], ci_ref[m_]], 1).astype(np.int32)
    # colored: the target's colour gradient as the library initialises it, fed to both sides
    tgt_c = R.initialize_pointcloud_for_colored_icp(cloud(tgt, tn, tc), 2 * EXACT_R)
    grad = tgt_c._color_gradient.cpu()
    ctx = R.IcpContext(cloud(src, None, sc), tgt_c, EXACT_R, R.TransformationEstimationForColoredICP())
    try:
        sums, ci = ctx.step(T)
    finally:
        ctx.close()
    np.testing.assert_array_equal(ci, ci_ref)
    ref = orc.jtj_jtr(orc.COLORED, P, tgt, corr, src_col=sc, tgt_nrm=tn, tgt_col=tc, tgt_grad=grad)
    sums_to_f32_equal(sums, ref, np.arange(28))
    assert sums[29] == len(corr)
    # GICP with general covariances (rotated with the source by the signed permutation: exactly)
    scov, tcov = _spd(rng, n), _spd(rng, m)
    ctx = R.IcpContext(cloud(src, cov=scov), cloud(tgt, cov=tcov), EXACT_R, R.TransformationEstimationForGeneralizedICP())
    try:
        sums, ci = ctx.step(T)
    finally:
        ctx.close()
    np.testing.assert_array_equal(ci, ci_ref)
    ref = orc.jtj_jtr(orc.GICP, P, tgt, corr, src_cov=orc.rotate_covariances(scov, T), tgt_cov=tcov)
    sums_to_f32_equal(sums, ref, np.arange(28))
    assert sums[29] == len(corr)


# ---- persistent ties through the whole loop -------------------------------------------------------------------------
KINDS = ["p2p", "p2plane", "symmetric", "colored", "gicp"]
TIE_R = 0.03


def _tie_clouds(dup_source):
    base, bn = datagen.surface(6000, 21)
    tgt, tn = features64.duplicated(base, bn, 22)
    tc = datagen.texture(tgt)
    gt = datagen.gt_transform((-0.6, 0.8, 1.2), (0.006, -0.004, 0.005))
    src, sn, sc = datagen.make_source(base, gt, 23, 24, 3e-4, attrs=[(bn, True), (datagen.texture(base), False)])
    if dup_source:  # the same seed repeats and shuffles rows identically: attributes stay with their points
        _, sc = features64.duplicated(src, sc, 25)
        src, sn = features64.duplicated(src, sn, 25)
    return src, sn, sc, tgt, tn, tc


def _run_device(kind, src, sn, sc, tgt, tn, tc, crit, r=TIE_R, init=None):
    init = np.eye(4) if init is None else init
    if kind == "p2p":
        return R.registration_icp(cloud(src), cloud(tgt), r, init, R.TransformationEstimationPointToPoint(), crit)
    if kind == "p2plane":
        return R.registration_icp(cloud(src), cloud(tgt, tn), r, init, R.TransformationEstimationPointToPlane(), crit)
    if kind == "symmetric":
        return R.registration_icp(cloud(src, sn), cloud(tgt, tn), r, init, R.TransformationEstimationSymmetricMethod(), crit)
    if kind == "colored":
        return R.registration_colored_icp(cloud(src, sn, sc), cloud(tgt, tn, tc), r, init, crit)
    return R.registration_generalized_icp(cloud(src, sn), cloud(tgt, tn), r, init, R.TransformationEstimationForGeneralizedICP(1e-3), crit)


def _run_oracle(orc, kind, src, sn, sc, tgt, tn, tc, crit, r=TIE_R, init=None, kdtree=False):
    kw = dict(init=init, relative_fitness=crit.relative_fitness, relative_rmse=crit.relative_rmse,
              max_iteration=crit.max_iteration, use_kdtree=kdtree)
    if kind == "p2p":
        return orc.registration_icp(orc.P2P, src, tgt, r, **kw)
    if kind == "p2plane":
        return orc.registration_icp(orc.P2PLANE, src, tgt, r, tgt_nrm=tn, **kw)
    if kind == "symmetric":
        return orc.registration_icp(orc.SYMMETRIC, src, tgt, r, src_nrm=sn, tgt_nrm=tn, **kw)
    if kind == "colored":
        nbr, _, _ = orc.search(tgt, tgt, 30, radius=2 * r, kdtree=True)
        grad = orc.color_gradient(tgt, tn, tc, nbr)
        return orc.registration_icp(orc.COLORED, src, tgt, r, src_col=sc, tgt_nrm=tn, tgt_col=tc, tgt_grad=grad, **kw)
    return orc.registration_icp(orc.GICP, src, tgt, r, src_cov=orc.covariances_from_normals(sn, 1e-3),
                                tgt_cov=orc.covariances_from_normals(tn, 1e-3), **kw)


def _first_twin(p):
    """for every row, the smallest row index holding the same point"""
    _, inv = np.unique(p, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    first = np.full(inv.max() + 1, len(p), np.int64)
    np.minimum.at(first, inv, np.arange(len(p)))
    return first[inv]


ENVS = ({"CPHB_CERT_GAIN": "0"}, {"CPHB_STATIC_SCHED": "0"}, {"CPHB_CERT_GAIN": "16", "CPHB_CERT_CAP": "4"})


def _env_runs_equal(monkeypatch, run, ref):
    """certificates off, the dynamic tile schedule, and far larger certificate margins: the same bits"""
    for env in ENVS:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        other = run()
        for k in env:
            monkeypatch.delenv(k)
        _same_bits(ref, other)


@pytest.mark.parametrize("dup_source", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_duplicate_targets_whole_loop(orc, monkeypatch, kind, dup_source):
    """every target point 2-3 times: each search ends on an exact tie, every iteration, and must pick the smaller-index
    twin like the brute-force oracle"""
    src, sn, sc, tgt, tn, tc = _tie_clouds(dup_source)
    assert 6000 <= len(src) <= 20000
    crit = R.ICPConvergenceCriteria(0, 0, 8)
    res = _run_device(kind, src, sn, sc, tgt, tn, tc, crit)
    ref = _run_oracle(orc, kind, src, sn, sc, tgt, tn, tc, crit)
    _compare(res, ref)
    assert res.fitness > 0.9
    j = res.correspondence_set[:, 1]
    first = _first_twin(tgt)
    np.testing.assert_array_equal(first[j], j)
    assert (np.bincount(first, minlength=len(tgt))[j] >= 2).all()  # every match had a twin to lose to
    _env_runs_equal(monkeypatch, lambda: _run_device(kind, src, sn, sc, tgt, tn, tc, crit), res)


def _half_tied_clouds():
    """half of the target points twice: a lane whose match has a twin is never certified (its second-nearest distance
    equals the nearest), the other half can be"""
    base, bn = datagen.surface(6000, 26)
    tgt = np.concatenate([base, base[:3000]])
    tn = np.concatenate([bn, bn[:3000]])
    perm = np.random.Generator(np.random.PCG64(27)).permutation(len(tgt))
    tgt, tn = np.ascontiguousarray(tgt[perm]), np.ascontiguousarray(tn[perm])
    src = datagen.make_source(base, datagen.gt_transform((-0.6, 0.8, 1.2), (0.006, -0.004, 0.005)), 28, 29, 3e-4)
    return src, tgt, tn


_CERT_SCRIPT = r"""
import sys
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import test_gpu_icp_edges as t
src, tgt, tn = t._half_tied_clouds()
res = t._run_device("p2plane", src, None, None, tgt, tn, None, t.R.ICPConvergenceCriteria(0, 0, 10))
print("fitness", res.fitness)
"""


def test_certificates_fire_under_ties(orc, monkeypatch):
    """the certificates are not merely harmless next to exact ties: they do skip searches there (CPHB_DEBUG_CERT is read
    once per process, so the counted run goes to a child process), and the loop still ends where the brute force does"""
    src, tgt, tn = _half_tied_clouds()
    crit = R.ICPConvergenceCriteria(0, 0, 10)
    res = _run_device("p2plane", src, None, None, tgt, tn, None, crit)
    _compare(res, _run_oracle(orc, "p2plane", src, None, None, tgt, tn, None, crit))
    j = res.correspondence_set[:, 1]
    twin = np.bincount(_first_twin(tgt), minlength=len(tgt))[_first_twin(tgt)] >= 2
    assert 0.3 < twin[j].mean() < 0.7                                   # both kinds of lanes are there
    np.testing.assert_array_equal(_first_twin(tgt)[j], j)
    _env_runs_equal(monkeypatch, lambda: _run_device("p2plane", src, None, None, tgt, tn, None, crit), res)
    env = dict(os.environ, CPHB_DEBUG_CERT="1")
    r = subprocess.run([sys.executable, "-c", _CERT_SCRIPT % (ROOT, os.path.join(ROOT, "tests"))], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stderr.splitlines()
    at = [i for i, s in enumerate(lines) if s.startswith("[cphb] certificates")]
    assert at, r.stderr[-2000:]
    counts = {int(a): int(b) for a, b in re.findall(r"(\d+)\*?:(\d+)/\d+", lines[at[-1] + 1])}
    assert set(range(11)) <= set(counts), lines[at[-1] + 1]
    assert sum(v for k, v in counts.items() if k >= 1) > 0, lines[at[-1] + 1]


# ---- degenerate clouds ----------------------------------------------------------------------------------------------
def _degenerate_cases():
    rng = np.random.Generator(np.random.PCG64(7))
    surf, sn = datagen.surface(3000, 8)
    one = np.array([[0.25, -0.5, 0.75]], np.float32)
    pile = np.concatenate([np.repeat(one, 2000, 0), one + rng.uniform(-0.02, 0.02, (6, 3)).astype(np.float32)])
    pile = pile[rng.permutation(len(pile))]
    line = np.zeros((2000, 3), np.float32)
    line[:, 0] = rng.permutation(2000).astype(np.float32) / np.float32(1024)
    line_n = np.tile(np.array([[0, 0, 1]], np.float32), (2000, 1))
    return {
        "single": (one + np.float32(0.004), one, np.array([[0, 0, 1]], np.float32)),
        "pile_target": ((pile[:500] + rng.normal(0, 0.005, (500, 3))).astype(np.float32), pile,
                        datagen.unit_normals(len(pile), 9)),
        "identical_source": (np.repeat(surf[1234:1235] + np.float32(0.003), 500, 0), surf, sn),
        "collinear_target": ((line[::3] + np.array([0.0004, 0.003, -0.002], np.float32)).astype(np.float32), line, line_n),
    }


@pytest.mark.parametrize("kind,case", [(k, c) for k in ("p2p", "p2plane")
                                        for c in ("single", "pile_target", "identical_source", "collinear_target")
                                        # identical sources make Kabsch's H rank 1 up to rounding: the rotation about
                                        # its axis is set by rounding noise, so only point-to-plane is comparable
                                        if (k, c) != ("p2p", "identical_source")])
def test_degenerate_clouds(orc, case, kind):
    src, tgt, tn = _degenerate_cases()[case]
    for crit in (R.ICPConvergenceCriteria(0, 0, 6), R.ICPConvergenceCriteria()):
        res = _run_device(kind, src, None, None, tgt, tn, None, crit, r=0.05)
        ref = _run_oracle(orc, kind, src, None, None, tgt, tn, None, crit, r=0.05, kdtree=True)
        _compare(res, ref)
        assert res.fitness > 0
        if kind == "p2p" and case == "single":
            # one correspondence: H = 0, and Kabsch (Eigen's SVD of a zero matrix) gives the identity rotation, so the
            # pose is a pure translation onto the target point
            np.testing.assert_array_equal(res.transformation[:3, :3], np.eye(3, dtype=np.float32))
            np.testing.assert_allclose(res.transformation[:3, 3], (tgt[0] - src[0]).astype(np.float64), atol=1e-7)


def test_planar_target_point_to_plane_is_singular(orc):
    """z = 0 target with normals +e_z: the J columns of rotation about z and of x / y translation are exactly 0, so
    the 6x6 system is exactly singular, the determinant test refuses it and every update is the identity"""
    rng = np.random.Generator(np.random.PCG64(12))
    tgt = np.zeros((5000, 3), np.float32)
    tgt[:, :2] = rng.random((5000, 2), dtype=np.float32)
    tn = np.tile(np.array([[0, 0, 1]], np.float32), (5000, 1))
    src = (tgt[rng.permutation(5000)[:3000]] + np.array([0.002, -0.001, 0.004], np.float32)).astype(np.float32)
    init = np.eye(4, dtype=np.float32)
    init[:3, 3] = [0.001, 0.0005, -0.002]
    for it in (1, 5):
        crit = R.ICPConvergenceCriteria(0, 0, it)
        res = R.registration_icp(cloud(src), cloud(tgt, tn), 0.02, init, R.TransformationEstimationPointToPlane(), crit)
        ref = orc.registration_icp(orc.P2PLANE, src, tgt, 0.02, init=init, tgt_nrm=tn, relative_fitness=0, relative_rmse=0,
                                   max_iteration=it)
        np.testing.assert_array_equal(res.transformation, init)
        _compare(res, ref)
    res = R.registration_icp(cloud(src), cloud(tgt, tn), 0.02, init, R.TransformationEstimationPointToPlane())
    np.testing.assert_array_equal(res.transformation, init)
    assert res.iterations == 1 and res.converged  # nothing moved: the first update already meets the criteria


@pytest.mark.parametrize("case", ["pile_target", "collinear_target"])
def test_search_on_degenerate_clouds(orc, case):
    """KDTreeFlann shares the ICP index build: zero-extent bounds (every point identical) and zero-width boxes (a line)"""
    src, tgt, _ = _degenerate_cases()[case]
    qry = np.concatenate([tgt[:300], src[:300]]).astype(np.float32)
    tree = cph.geometry.KDTreeFlann(cph.geometry.PointCloud(tgt))
    for k, radius in ((1, None), (7, None), (40, None), (16, 0.01), (50, 0.05)):
        if radius is None:
            cnt, idx, d2 = tree.search_knn(qry, k)
            oi, od, oc = orc.search(tgt, qry, k, kdtree=False)
        else:
            cnt, idx, d2 = tree.search_radius(qry, radius, k)
            oi, od, oc = orc.search(tgt, qry, k, radius=radius, kdtree=False)
        assert cnt == oc
        np.testing.assert_array_equal(idx.cpu(), oi)
        np.testing.assert_array_equal(d2.cpu().view(np.uint32), od.view(np.uint32))


# ---- past the 1 M-point shapes --------------------------------------------------------------------------------------
def test_icp_p2plane_past_1m(orc, monkeypatch):
    """1.1 M-point target (index depth top = 3) and 1.1 M-point source (two correspondence compaction chunks); every
    warp claims several tiles under both schedules"""
    n = 1_100_000
    tgt, tn = datagen.surface(n, 41)
    src = datagen.make_source(tgt, datagen.gt_transform((-1.0, 1.5, 2.0), (0.01, -0.005, 0.008)), 42, 43, 5e-4)
    crit = R.ICPConvergenceCriteria(0, 0, 10)

    def run():
        return R.registration_icp(cloud(src), cloud(tgt, tn), 0.02, np.eye(4), R.TransformationEstimationPointToPlane(), crit)

    res = run()
    ref = orc.registration_icp(orc.P2PLANE, src, tgt, 0.02, tgt_nrm=tn, relative_fitness=0, relative_rmse=0, max_iteration=10)
    _compare(res, ref)
    assert res.fitness > 0.9
    for env in ENVS[:2]:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        other = run()
        for k in env:
            monkeypatch.delenv(k)
        _same_bits(res, other)


def test_evaluate_registration_three_chunks(orc):
    """2.5 M sources: the compaction scan carries its running offset across three chunks of 1024 blocks"""
    tgt = datagen.surface(1_100_000, 44)[0]
    src = datagen.surface(2_500_000, 45)[0]
    T = np.eye(4, dtype=np.float32)
    T[:3, 3] = [0.0003, -0.0002, 0.0]
    res = R.evaluate_registration(cloud(src), cloud(tgt), 0.0007, T)
    corr, fit, rmse = orc.correspondences(orc.transform_points(src, T), tgt, 0.0007)
    assert 0.05 < fit < 0.95                       # gaps: later chunks' offsets differ from their first index
    np.testing.assert_array_equal(res.correspondence_set, corr)
    assert abs(res.fitness - fit) < 1e-7 and abs(res.inlier_rmse - rmse) < 1e-7


# ---- loop stop rules ------------------------------------------------------------------------------------------------
def _stop_pair():
    tgt, tn = datagen.surface(8000, 51)
    gt = datagen.gt_transform((-1.0, 1.5, 2.0), (0.01, -0.005, 0.008))
    src, sn, sc = datagen.make_source(tgt, gt, 52, 53, 5e-4, attrs=[(tn, True), (datagen.texture(tgt), False)])
    return src, sn, sc, tgt, tn, datagen.texture(tgt)


FAR = np.eye(4, dtype=np.float32)
FAR[:3, 3] = [100.0, 0.0, 0.0]
STOP_CASES = {
    "max_iteration_0": (0.03, None, (0, 0, 0)),
    "max_iteration_1": (0.03, None, (0, 0, 1)),
    "stops_at_first_update": (0.03, None, (1.0, 1.0, 30)),
    "stops_after_a_few": (0.03, None, (1e-3, 1e-3, 30)),
    "radius_matches_nothing": (1e-7, None, (1e-6, 1e-6, 30)),
    "init_out_of_range": (0.03, FAR, (1e-6, 1e-6, 30)),
}


@pytest.mark.parametrize("case", sorted(STOP_CASES))
@pytest.mark.parametrize("kind", ["p2p", "p2plane", "symmetric"])
def test_stop_rules(orc, case, kind):
    src, sn, sc, tgt, tn, tc = _stop_pair()
    r, init, c = STOP_CASES[case]
    crit = R.ICPConvergenceCriteria(*c)
    res = _run_device(kind, src, sn, sc, tgt, tn, tc, crit, r=r, init=init)
    ref = _run_oracle(orc, kind, src, sn, sc, tgt, tn, tc, crit, r=r, init=init, kdtree=True)
    _compare(res, ref)
    assert res.converged == (ref["iterations"] < crit.max_iteration)
    if case == "stops_after_a_few":
        assert 1 < ref["iterations"] < crit.max_iteration
    if case == "stops_at_first_update":
        assert ref["iterations"] == 1
    # no correspondence: every update is the identity (for point-to-point: Kabsch of H = 0, Eigen's SVD gives U = V = I)
    if case in ("radius_matches_nothing", "init_out_of_range"):
        assert res.fitness == 0 and len(res.correspondence_set) == 0
        np.testing.assert_array_equal(res.transformation, np.eye(4, dtype=np.float32) if init is None else init)


@pytest.mark.parametrize("missing", ["symmetric_source_normals", "p2plane_target_normals", "colored_source_colors",
                                     "gicp_covariances"])
def test_missing_attribute_is_identity(orc, missing):
    """an estimator whose attribute is missing leaves every update the identity, as the reference does"""
    src, sn, sc, tgt, tn, tc = _stop_pair()
    crit = R.ICPConvergenceCriteria(1e-6, 1e-6, 5)
    init = datagen.gt_transform((-0.2, 0.1, 0.3), (0.002, 0.0, -0.001)).astype(np.float32)
    kw = dict(init=init, relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=5)
    if missing == "symmetric_source_normals":
        res = R.registration_icp(cloud(src), cloud(tgt, tn), 0.03, init, R.TransformationEstimationSymmetricMethod(), crit)
        ref = orc.registration_icp(orc.SYMMETRIC, src, tgt, 0.03, tgt_nrm=tn, **kw)
    elif missing == "p2plane_target_normals":
        res = R.registration_icp(cloud(src), cloud(tgt), 0.03, init, R.TransformationEstimationPointToPlane(), crit)
        ref = orc.registration_icp(orc.P2PLANE, src, tgt, 0.03, **kw)
    elif missing == "colored_source_colors":
        res = R.registration_colored_icp(cloud(src, sn), cloud(tgt, tn, tc), 0.03, init, crit)
        ref = orc.registration_icp(orc.COLORED, src, tgt, 0.03, tgt_nrm=tn, tgt_col=tc,
                                   tgt_grad=np.zeros_like(tgt), **kw)
    else:
        res = R.registration_icp(cloud(src), cloud(tgt), 0.03, init, R.TransformationEstimationForGeneralizedICP(), crit)
        ref = orc.registration_icp(orc.GICP, src, tgt, 0.03, **kw)
    _compare(res, ref)
    np.testing.assert_array_equal(res.transformation, init)
    assert res.iterations == 1 and res.converged
