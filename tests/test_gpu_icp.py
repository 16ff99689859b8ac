"""GPU parity: fused ICP iteration / RegistrationICP (C ABI through the Python mirror) vs the CPU oracle.

Per step (same pose in, oracle correspondences vs kernel correspondences): indices bit-exact,
the 27 normal-equation sums equal after rounding to float32 (both sides accumulate exact products
in float64).  Whole loop: final pose within 1e-5 Frobenius (north_star), fitness / rmse to 1e-6,
correspondence sets identical.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cupoch_b200 as cph
from cupoch_b200.testing import datagen

R = cph.registration
POSE_TOL = 1e-5  # Frobenius, BASELINE.json north_star


def cloud(p, n=None, c=None, cov=None):
    pc = cph.geometry.PointCloud(p)
    if n is not None:
        pc.normals = n
    if c is not None:
        pc.colors = c
    if cov is not None:
        pc.covariances = cov
    return pc


def small_pair(n=20000, sigma=5e-4, surface=True):
    if surface:
        tgt, tn = datagen.surface(n, 11)
    else:
        tgt, tn = datagen.uniform_cube(n, 1), datagen.unit_normals(n, 12)
    src, sn = datagen.make_source(tgt, datagen.gt_transform((-1.0, 1.5, 2.0), (0.01, -0.005, 0.008)), 13, 14, sigma,
                                  attrs=[(tn, True)])
    return src, sn, tgt, tn


def sums_to_f32_equal(a, b, idx):
    a32, b32 = a[idx].astype(np.float32), b[idx].astype(np.float32)
    # both are float64 sums of identical exact products in different orders: equal to ~1e-13 relative,
    # i.e. identical after float32 rounding except on a rounding boundary (<= 1 ulp)
    np.testing.assert_allclose(a[idx], b[idx], rtol=1e-10, atol=1e-12 * np.abs(a[idx]).max())
    assert (np.abs(a32.view(np.int32) - b32.view(np.int32)) <= 1).all()


@pytest.mark.parametrize("surface", [True, False])
def test_step_p2plane(orc, surface):
    src, sn, tgt, tn = small_pair(surface=surface)
    ctx = R.IcpContext(cloud(src), cloud(tgt, tn), 0.03, R.TransformationEstimationPointToPlane())
    for T in (np.eye(4, dtype=np.float32), datagen.gt_transform((-0.5, 1.0, 1.0), (0.005, 0, 0.004)).astype(np.float32)):
        sums, ci = ctx.step(T)
        moved = orc.transform_points(src, T)
        corr, fit, rmse = orc.correspondences(moved, tgt, 0.03)
        ref = np.full(len(src), -1, np.int32)
        ref[corr[:, 0]] = corr[:, 1]
        np.testing.assert_array_equal(ci, ref)                       # indices bit-exact
        osums = orc.jtj_jtr(orc.P2PLANE, moved, tgt, corr, tgt_nrm=tn)
        sums_to_f32_equal(sums, osums, np.arange(28))
        assert sums[29] == len(corr)
    ctx.close()


def test_step_p2p(orc):
    src, sn, tgt, tn = small_pair()
    ctx = R.IcpContext(cloud(src), cloud(tgt), 0.03, R.TransformationEstimationPointToPoint())
    T = np.eye(4, dtype=np.float32)
    sums, ci = ctx.step(T)
    corr, _, _ = orc.correspondences(src, tgt, 0.03)
    _, S = orc.kabsch(src, tgt, corr)
    sums_to_f32_equal(sums, S, np.arange(15))
    assert sums[29] == len(corr) == S[15]
    ctx.close()


def _compare(res, ref, pose_tol=POSE_TOL, exact_corr=True):
    d = np.linalg.norm(res.transformation.astype(np.float64) - ref["transformation"].astype(np.float64))
    assert d <= pose_tol, "pose differs by %g (Frobenius)" % d
    assert res.iterations == ref["iterations"]
    assert abs(res.fitness - ref["fitness"]) <= 1e-6
    assert abs(res.inlier_rmse - ref["inlier_rmse"]) <= 1e-6
    if exact_corr:
        np.testing.assert_array_equal(res.correspondence_set, ref["correspondence_set"])
    else:
        a = {tuple(x) for x in res.correspondence_set.tolist()}
        b = {tuple(x) for x in ref["correspondence_set"].tolist()}
        assert len(a ^ b) <= max(2, len(b) // 5000), "correspondence sets differ in %d pairs" % len(a ^ b)
    return d


def _check_icp_p2plane(orc, n, iterations):
    src, sn, tgt, tn = small_pair(n=n)
    crit = R.ICPConvergenceCriteria(0, 0, iterations)
    res = R.registration_icp(cloud(src), cloud(tgt, tn), 0.03, np.eye(4), R.TransformationEstimationPointToPlane(), crit)
    ref = orc.registration_icp(orc.P2PLANE, src, tgt, 0.03, tgt_nrm=tn, relative_fitness=0, relative_rmse=0,
                               max_iteration=iterations)
    _compare(res, ref)
    gt = datagen.gt_transform((-1.0, 1.5, 2.0), (0.01, -0.005, 0.008))
    assert np.linalg.norm(res.transformation - gt) < 2e-3   # and it actually registers
    assert res.fitness > 0.99


def test_icp_p2plane(orc):
    _check_icp_p2plane(orc, 20000, 12)


def test_icp_p2plane_30k(orc):
    """A larger cloud and a longer run (30 000 points, 14 iterations) on the default path, against the same oracle."""
    _check_icp_p2plane(orc, 30000, 14)


def test_icp_p2plane_init_and_convergence(orc):
    src, sn, tgt, tn = small_pair(sigma=0.0)
    init = datagen.gt_transform((-0.9, 1.4, 1.9), (0.009, -0.004, 0.007)).astype(np.float32)
    crit = R.ICPConvergenceCriteria(1e-6, 1e-6, 30)
    res = R.registration_icp(cloud(src), cloud(tgt, tn), 0.03, init, R.TransformationEstimationPointToPlane(), crit)
    ref = orc.registration_icp(orc.P2PLANE, src, tgt, 0.03, init=init, tgt_nrm=tn)
    assert ref["iterations"] < 30 and res.converged          # stopped by the criteria, like the oracle
    _compare(res, ref)


def test_icp_p2p(orc):
    src, sn, tgt, tn = small_pair(surface=False)
    crit = R.ICPConvergenceCriteria(0, 0, 15)
    res = R.registration_icp(cloud(src), cloud(tgt), 0.05, np.eye(4), R.TransformationEstimationPointToPoint(), crit)
    ref = orc.registration_icp(orc.P2P, src, tgt, 0.05, relative_fitness=0, relative_rmse=0, max_iteration=15)
    _compare(res, ref)


def test_icp_symmetric(orc):
    src, sn, tgt, tn = small_pair()
    crit = R.ICPConvergenceCriteria(0, 0, 8)
    res = R.registration_icp(cloud(src, sn), cloud(tgt, tn), 0.03, np.eye(4), R.TransformationEstimationSymmetricMethod(), crit)
    ref = orc.registration_icp(orc.SYMMETRIC, src, tgt, 0.03, src_nrm=sn, tgt_nrm=tn, relative_fitness=0, relative_rmse=0,
                               max_iteration=8)
    _compare(res, ref)


def test_icp_generalized(orc):
    src, sn, tgt, tn = small_pair(n=12000)
    crit = R.ICPConvergenceCriteria(0, 0, 8)
    res = R.registration_generalized_icp(cloud(src, sn), cloud(tgt, tn), 0.03, np.eye(4),
                                         R.TransformationEstimationForGeneralizedICP(1e-3), crit)
    scov, tcov = orc.covariances_from_normals(sn, 1e-3), orc.covariances_from_normals(tn, 1e-3)
    ref = orc.registration_icp(orc.GICP, src, tgt, 0.03, src_cov=scov, tgt_cov=tcov, relative_fitness=0, relative_rmse=0,
                               max_iteration=8)
    # FastEigen3x3's acos / cos are a shared deterministic specification (oracle.c "deterministic acos / cos"), so GICP
    # is bit-reproducible like the other estimators: identical correspondence sets
    _compare(res, ref)


def test_icp_colored(orc):
    n = 15000
    tgt, tn = datagen.surface(n, 31)
    tc = datagen.texture(tgt)
    gt = datagen.gt_transform((-0.4, 0.6, 0.8), (0.004, -0.003, 0.002))
    src, sn, sc = datagen.make_source(tgt, gt, 33, 34, 2e-4, attrs=[(tn, True), (tc, False)])
    crit = R.ICPConvergenceCriteria(0, 0, 8)
    r = 0.03
    res = R.registration_colored_icp(cloud(src, sn, sc), cloud(tgt, tn, tc), r, np.eye(4), crit)
    nbr, _, _ = orc.search(tgt, tgt, 30, radius=2 * r, kdtree=True)
    grad = orc.color_gradient(tgt, tn, tc, nbr)
    ref = orc.registration_icp(orc.COLORED, src, tgt, r, src_col=sc, tgt_nrm=tn, tgt_col=tc, tgt_grad=grad,
                               relative_fitness=0, relative_rmse=0, max_iteration=8)
    _compare(res, ref)


def test_evaluate_registration(orc):
    src, sn, tgt, tn = small_pair()
    T = datagen.gt_transform((-1.0, 1.5, 2.0), (0.01, -0.005, 0.008)).astype(np.float32)
    res = R.evaluate_registration(cloud(src), cloud(tgt), 0.01, T)
    corr, fit, rmse = orc.correspondences(orc.transform_points(src, T), tgt, 0.01)
    np.testing.assert_array_equal(res.correspondence_set, corr)
    assert abs(res.fitness - fit) < 1e-7 and abs(res.inlier_rmse - rmse) < 1e-7


def test_degenerate_inputs(orc):
    src, sn, tgt, tn = small_pair(n=3000)
    # max_correspondence_distance <= 0: the reference logs and returns fitness 0 / empty set (registration.cu:40-42)
    res = R.registration_icp(cloud(src), cloud(tgt, tn), 0.0, np.eye(4), R.TransformationEstimationPointToPlane())
    assert res.fitness == 0 and len(res.correspondence_set) == 0
    np.testing.assert_array_equal(res.transformation, np.eye(4, dtype=np.float32))
    # point-to-plane without target normals: update is identity, loop converges immediately
    res = R.registration_icp(cloud(src), cloud(tgt), 0.03, np.eye(4), R.TransformationEstimationPointToPlane())
    np.testing.assert_array_equal(res.transformation, np.eye(4, dtype=np.float32))
    assert res.fitness > 0
    # tiny clouds
    res = R.registration_icp(cloud(src[:5]), cloud(tgt[:7], tn[:7]), 10.0, np.eye(4), R.TransformationEstimationPointToPlane())
    ref = orc.registration_icp(orc.P2PLANE, src[:5], tgt[:7], 10.0, tgt_nrm=tn[:7])
    assert res.iterations == ref["iterations"]


def test_icp_1m_properties():
    """Full-size (config 2) properties that need no oracle: converges to the known pose, every
    iteration deterministic run-to-run (bitwise)."""
    n = 1_000_000
    tgt, tn = datagen.surface(n, 11)
    gt = datagen.gt_transform()
    src = datagen.make_source(tgt, gt, 13, 14, 5e-4)
    ctx = R.IcpContext(cloud(src), cloud(tgt, tn), 0.02, R.TransformationEstimationPointToPlane(), R.ICPConvergenceCriteria(0, 0, 30))
    a = ctx.run(np.eye(4))
    b = ctx.run(np.eye(4))
    np.testing.assert_array_equal(a.transformation, b.transformation)
    np.testing.assert_array_equal(a.correspondence_set, b.correspondence_set)
    assert a.iterations == 30
    assert np.linalg.norm(a.transformation - gt) < 5e-3
    assert a.fitness > 0.95
    i, j = a.correspondence_set[:, 0], a.correspondence_set[:, 1]
    assert (np.diff(i) > 0).all() and j.min() >= 0 and j.max() < n          # ascending in i, valid j
    ctx.close()


def test_kabsch_golden(golden, orc):
    """tests/registration/kabsch.cpp:35-55: a 30-degree z rotation is recovered (isApprox 1e-3)."""
    g = golden["kabsch"]
    p = np.array(g["points"], np.float32)
    a = np.deg2rad(np.float32(g["angle_deg_z"]))
    T = np.array([[np.cos(a), -np.sin(a), 0, 0], [np.sin(a), np.cos(a), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)
    q = orc.transform_points(p, T)
    Rk = R.kabsch(p, q)
    assert np.linalg.norm(Rk - T) <= g["tolerance"] * min(np.linalg.norm(Rk), np.linalg.norm(T))
    corr = np.stack([np.arange(len(p)), np.arange(len(p))], 1).astype(np.int32)
    To, _ = orc.kabsch(p, q, corr)
    np.testing.assert_array_equal(Rk, To)      # same double-precision SVD path, bit for bit


def test_compute_transformation_and_rmse(orc):
    """TransformationEstimation*::ComputeTransformation / ComputeRMSE on an explicit correspondence list."""
    src, sn, tgt, tn = small_pair(n=8000)
    corr, _, _ = orc.correspondences(src, tgt, 0.03)
    s_pc, t_pc = cloud(src, sn), cloud(tgt, tn)
    # point to plane
    est = R.TransformationEstimationPointToPlane()
    sums = orc.jtj_jtr(orc.P2PLANE, src, tgt, corr, tgt_nrm=tn)
    ok, To = orc.solve_jtj(sums[:21].astype(np.float32), sums[21:27].astype(np.float32))
    np.testing.assert_array_equal(est.compute_transformation(s_pc, t_pc, corr), To)
    assert abs(est.compute_rmse(s_pc, t_pc, corr) - np.sqrt(np.float32(sums[27]) / np.float32(len(corr)))) < 1e-7
    # point to point (Kabsch with the divide-by-N quirk) and its rmse
    est = R.TransformationEstimationPointToPoint()
    To, _ = orc.kabsch(src, tgt, corr)
    np.testing.assert_array_equal(est.compute_transformation(cloud(src), cloud(tgt), corr), To)
    d = src[corr[:, 0]].astype(np.float64) - tgt[corr[:, 1]]
    assert abs(est.compute_rmse(cloud(src), cloud(tgt), corr) - np.sqrt((d ** 2).sum() / len(corr))) < 1e-6
    # empty correspondence set -> identity (transformation_estimation.cu:199-200)
    np.testing.assert_array_equal(R.TransformationEstimationPointToPlane().compute_transformation(s_pc, t_pc, np.zeros((0, 2), np.int32)),
                                  np.eye(4, dtype=np.float32))


def test_gicp_nonfinite_rows_are_dropped(orc):
    """Covariances whose degenerate eigen-plane is axis aligned make the reference's FastEigen3x3 evaluate
    signf(0) = 0/0 (eigenvalue.inl:28): every GICP row is NaN there.  Product and oracle drop such rows
    (DESIGN.md parity hazard 8) instead of returning an all-NaN pose."""
    rng = np.random.default_rng(5)
    n = 6000
    nrm = np.array([1.0, 1.0, 0.0]) / np.sqrt(2.0)
    uv = rng.random((n, 2))
    tgt = (np.outer(uv[:, 0], [1, -1, 0]) / np.sqrt(2) + np.outer(uv[:, 1], [0, 0, 1])).astype(np.float32)
    src = (tgt[rng.permutation(n)] + 0.002 * nrm).astype(np.float32)
    nn = np.tile(nrm.astype(np.float32), (n, 1))
    crit = R.ICPConvergenceCriteria(0, 0, 3)
    res = R.registration_generalized_icp(cloud(src, nn), cloud(tgt, nn), 0.01, np.eye(4), None, crit)
    cov = orc.covariances_from_normals(nn, 1e-3)
    ref = orc.registration_icp(orc.GICP, src, tgt, 0.01, src_cov=cov, tgt_cov=cov, relative_fitness=0, relative_rmse=0, max_iteration=3)
    assert np.isfinite(res.transformation).all() and np.isfinite(ref["transformation"]).all()
    assert res.fitness > 0.5
    _compare(res, ref)


def test_user_defined_estimator_generic_loop(orc):
    """A Python subclass of TransformationEstimation (what the reference's trampoline, registration.cpp:36-60, allows)
    runs the reference's generic loop (registration.cu:145-172): with an estimator that delegates to the built-in
    point-to-plane solve it must end exactly where the fused path and the oracle end."""
    src, sn, tgt, tn = small_pair()

    class Mine(R.TransformationEstimation):   # type stays Unspecified
        calls = 0

        def compute_transformation(self, source, target, corres):
            Mine.calls += 1
            assert corres.dtype == np.int32 and corres.shape[1] == 2
            return R.TransformationEstimationPointToPlane().compute_transformation(source, target, corres)

    init = datagen.gt_transform((-0.3, 0.2, 0.4), (0.002, 0.0, -0.001)).astype(np.float32)
    crit = R.ICPConvergenceCriteria(0, 0, 6)
    res = R.registration_icp(cloud(src), cloud(tgt, tn), 0.03, init, Mine(), crit)
    ref = orc.registration_icp(orc.P2PLANE, src, tgt, 0.03, init=init, tgt_nrm=tn, relative_fitness=0, relative_rmse=0, max_iteration=6)
    assert Mine.calls == 6
    _compare(res, ref)
    fused = R.registration_icp(cloud(src), cloud(tgt, tn), 0.03, init, R.TransformationEstimationPointToPlane(), crit)
    # (the standalone ComputeTransformation adds its float64 products in another order than the fused kernel: the
    # poses agree to the last bits, not necessarily in them)
    assert np.linalg.norm(res.transformation.astype(np.float64) - fused.transformation) <= POSE_TOL
    np.testing.assert_array_equal(res.correspondence_set, fused.correspondence_set)
    # host-buffer entry point takes the same route
    res_h = R.registration_icp_host(src, tgt, 0.03, init, Mine(), crit, target_normals=tn, return_correspondences=True)
    np.testing.assert_array_equal(res_h.transformation, res.transformation)


def test_create_checks_shard_rank_before_any_work():
    """an out-of-range shard rank is refused with the other argument checks: no source ordering, no index build, no
    launch"""
    import ctypes as C
    L = cph._lib.lib()
    src, sn, tgt, tn = small_pair(2000)
    s, t = cloud(src), cloud(tgt)
    p = R._params(R.TransformationEstimationPointToPoint(), 0.03, R.ICPConvergenceCriteria(), shard=(5, 2))
    sc, tc = s._cloud(), t._cloud()
    h = C.c_void_p()
    before = L.cphb_launch_count()
    rc = L.cphb_icp_create(C.byref(sc), C.byref(tc), C.byref(p), None, C.byref(h))
    assert rc == cph._lib.CPHB_ERR_INVALID
    assert "shard_rank 5 outside [0,2)" in L.cphb_last_error().decode()
    assert L.cphb_launch_count() == before and not h.value


@pytest.mark.parametrize("close_first", [0, 1])
def test_two_live_contexts_match_a_lone_one(close_first):
    """the second live context on a thread has its own pinned staging: both give a lone context's bits, whichever
    is closed first"""
    src, sn, tgt, tn = small_pair()
    init = datagen.gt_transform((-0.3, 0.2, 0.4), (0.002, 0.0, -0.001)).astype(np.float32)
    crit = R.ICPConvergenceCriteria(0, 0, 12)
    make = lambda: R.IcpContext(cloud(src), cloud(tgt, tn), 0.03, R.TransformationEstimationPointToPlane(), crit)
    lone = make()
    ref = lone.run(init)
    ref_step = lone.step(init)
    lone.close()
    ctx = [make(), make()]
    try:
        for c in ctx:
            r = c.run(init)
            np.testing.assert_array_equal(r.transformation, ref.transformation)
            np.testing.assert_array_equal(r.correspondence_set, ref.correspondence_set)
            assert (r.iterations, r.fitness, r.inlier_rmse) == (ref.iterations, ref.fitness, ref.inlier_rmse)
        ctx[close_first].close()
        other = ctx[1 - close_first]
        sums, ci = other.step(init)
        np.testing.assert_array_equal(sums, ref_step[0])
        np.testing.assert_array_equal(ci, ref_step[1])
        r = other.run(init)
        np.testing.assert_array_equal(r.transformation, ref.transformation)
        again = make()  # takes over whatever staging the closed context released
        try:
            np.testing.assert_array_equal(again.run(init).transformation, ref.transformation)
        finally:
            again.close()
    finally:
        for c in ctx:
            c.close()
