"""The device ICP estimators against the float64 restatement of cupoch_b200/testing/icp64.py, within its bounds: the
standalone ComputeTransformation / ComputeRMSE (estimate_kernel, estimate_solve_kernel, cphb_compute_rmse) for all five
estimators at correspondence counts either side of the 256-thread block and up to 10^6, with missing attributes and
lambda_geometric at its edges; the fused step's sums (IcpContext.step); and a replay of the loop, each update of a run
against the restated update of the source at the pose before it, composed on the left."""
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cupoch_b200 as cph
from cupoch_b200.testing import datagen, icp64
from cupoch_b200.utility import DeviceArray

R = cph.registration
U = icp64.U
KINDS = {"p2p": icp64.P2P, "p2plane": icp64.P2PLANE, "symmetric": icp64.SYMMETRIC, "colored": icp64.COLORED,
         "gicp": icp64.GICP}
COUNTS = [1, 255, 256, 257, 2049, 1_000_000]
STATS = {}  # estimator -> largest observed deviation as a fraction of its bound (printed)
MUTANT_MARGIN = 10.0  # a mutant's pose must be at least this many bounds away


def _frac(d, bound):
    return 0.0 if d == 0 else d / bound


def _note(kind, what, ratio):
    key = "%s %s" % (kind, what)
    STATS[key] = max(STATS.get(key, 0.0), float(ratio))
    print("%s: %.3g of the bound" % (key, ratio))
    assert ratio <= 1.0, key


def cloud(p, n=None, c=None, cov=None, grad=None):
    pc = cph.geometry.PointCloud(p)
    if n is not None:
        pc.normals = n
    if c is not None:
        pc.colors = c
    if cov is not None:
        pc.covariances = cov
    if grad is not None:
        pc._color_gradient = DeviceArray.wrap(np.ascontiguousarray(grad, np.float32))
    return pc


def estimation(kind, lam=0.968):
    return {"p2p": R.TransformationEstimationPointToPoint, "p2plane": R.TransformationEstimationPointToPlane,
            "symmetric": R.TransformationEstimationSymmetricMethod, "gicp": R.TransformationEstimationForGeneralizedICP,
            "colored": lambda: R.TransformationEstimationForColoredICP(lam)}[kind]()


@functools.lru_cache(None)
def big_scene():
    """10^6 target points, the source their permutation moved by a small pose plus noise: correspondence k is
    (k, perm[k]) with no search.  The colour gradient is an input here, any field will do."""
    from oracle import oracle_py as orc
    n = 1_000_000
    tgt, tn = datagen.surface(n, 61)
    tc = datagen.texture(tgt)
    gt = datagen.gt_transform((-0.4, 0.6, 0.8), (0.004, -0.003, 0.002))
    src, sn, sc = datagen.make_source(tgt, gt, 62, 63, 3e-4, attrs=[(tn, True), (tc, False)])
    perm = np.random.Generator(np.random.PCG64(62)).permutation(n)
    corr = np.stack([np.arange(n), perm], 1).astype(np.int32)
    grad = (0.3 * datagen.unit_normals(n, 64)).astype(np.float32)
    # GICP: source covariances from normals independent of the target's.  With nearly parallel normals (the loop scenes
    # below) the two tangential eigenvalues of W^2 meet, FastEigen3x3's acos term saturates at about lam2 sqrt(U) per row
    # and the worst-case pose bound is no longer small against the update; here the bound pins the pose
    attrs = dict(src_nrm=sn, src_col=sc, src_cov=orc.covariances_from_normals(datagen.unit_normals(n, 65), 1e-3),
                 tgt_nrm=tn, tgt_col=tc, tgt_grad=grad, tgt_cov=orc.covariances_from_normals(tn, 1e-3))
    return src, tgt, corr, attrs


def _clouds(kind, src, tgt, a):
    if kind == "p2p":
        return cloud(src), cloud(tgt)
    if kind == "p2plane":
        return cloud(src), cloud(tgt, a["tgt_nrm"])
    if kind == "symmetric":
        return cloud(src, a["src_nrm"]), cloud(tgt, a["tgt_nrm"])
    if kind == "colored":
        return cloud(src, c=a["src_col"]), cloud(tgt, a["tgt_nrm"], a["tgt_col"], grad=a["tgt_grad"])
    return cloud(src, cov=a["src_cov"]), cloud(tgt, cov=a["tgt_cov"])


def _restated(kind, src, tgt, corr, a, lam=0.968, src_err=0.0, det_thresh=1e-6):
    """-> (update T, Frobenius bound, gate decision firm)"""
    k = KINDS[kind]
    if k == icp64.P2P:
        T, err = icp64.kabsch(src, tgt, corr, len(src), src_err=src_err)
        return T, err, True
    keys = {"p2plane": ("tgt_nrm",), "symmetric": ("src_nrm", "tgt_nrm"),
            "colored": ("src_col", "tgt_nrm", "tgt_col", "tgt_grad"), "gicp": ("src_cov", "tgt_cov")}[kind]
    ne = icp64.normal_equations(k, src, tgt, corr, lambda_geometric=lam, src_err=src_err, **{x: a[x] for x in keys})
    sv = icp64.solve(k, ne["S"], ne["bound"], det_thresh)
    return sv["T"], sv["err"], sv["firm"]


def _rmse(kind, src, tgt, corr, a, lam=0.968):
    keys = {"p2p": (), "p2plane": ("tgt_nrm",), "symmetric": ("src_nrm", "tgt_nrm"),
            "colored": ("src_col", "tgt_nrm", "tgt_col", "tgt_grad"), "gicp": ("src_cov", "tgt_cov")}[kind]
    return icp64.rmse(KINDS[kind], src, tgt, corr, lambda_geometric=lam, **{x: a[x] for x in keys})


# ---- standalone ComputeTransformation / ComputeRMSE ----------------------------------------------------------------
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_standalone(kind, count):
    src, tgt, corr_all, a = big_scene()
    corr = np.ascontiguousarray(corr_all[np.linspace(0, len(corr_all) - 1, count).astype(np.int64)])
    s_pc, t_pc = _clouds(kind, src, tgt, a)
    lams = [0.0, 0.25, 1.0] if kind == "colored" and count == 2049 else [0.968]
    for lam in lams:
        est = estimation(kind, lam)
        r = est.compute_rmse(s_pc, t_pc, corr)
        r64, rerr = _rmse(kind, src, tgt, corr, a, lam)
        _note(kind, "compute_rmse", _frac(abs(r - r64), rerr))
        T = est.compute_transformation(s_pc, t_pc, corr).astype(np.float64)
        T64, err, firm = _restated(kind, src, tgt, corr, a, lam)
        assert firm, "the gate's decision is within its margin"  # (never the case on these inputs)
        _note(kind, "compute_transformation", _frac(np.linalg.norm(T - T64), err))
        if count >= 255 and not np.array_equal(T64, np.eye(4)):
            # a full-rank system: the bound must be small against the update it checks, or the check says nothing
            # (photometric rows alone, lambda = 0, constrain the pose weakly: kappa(A) is larger, so 0.3 there)
            frac = 0.3 if kind == "colored" and lam == 0.0 else 0.1
            print("%s %d lambda %g: pose bound %.3g of the update" % (kind, count, lam, err / np.linalg.norm(T64 - np.eye(4))))
            assert err <= frac * np.linalg.norm(T64 - np.eye(4))


@pytest.mark.parametrize("missing", ["p2plane_target_normals", "symmetric_source_normals", "colored_target_gradient",
                                     "colored_source_colors", "gicp_covariances"])
def test_standalone_missing_attribute(missing):
    """an estimator without an attribute it needs returns the identity and an RMSE of 0"""
    src, tgt, corr_all, a = big_scene()
    corr = np.ascontiguousarray(corr_all[:2049])
    kind = missing.split("_")[0]
    s_pc, t_pc = {
        "p2plane_target_normals": lambda: (cloud(src), cloud(tgt)),
        "symmetric_source_normals": lambda: (cloud(src), cloud(tgt, a["tgt_nrm"])),
        "colored_target_gradient": lambda: (cloud(src, c=a["src_col"]), cloud(tgt, a["tgt_nrm"], a["tgt_col"])),
        "colored_source_colors": lambda: (cloud(src), cloud(tgt, a["tgt_nrm"], a["tgt_col"], grad=a["tgt_grad"])),
        "gicp_covariances": lambda: (cloud(src), cloud(tgt)),
    }[missing]()
    est = estimation(kind)
    np.testing.assert_array_equal(est.compute_transformation(s_pc, t_pc, corr), np.eye(4, dtype=np.float32))
    # every row needs the missing attribute (icp_rows.cuh, load_tgt_orig), so every row and every RMSE term is zero
    assert est.compute_rmse(s_pc, t_pc, corr) == 0.0


# ---- fused step and loop replay ------------------------------------------------------------------------------------
@functools.lru_cache(None)
def loop_scene(scene=None):
    """a 20 000-point surface pair; scene="cone" turns it so that the flat parts' normals lie inside GICP's -e1 cone.
    scene="colored" is the 15 000-point pair of test_gpu_icp.py::test_icp_colored, whose fitted colour gradient keeps the
    colored loop converging at lambda = 0.5 (on the 20 000-point pair its outliers, up to 1e5, make it diverge)"""
    if scene == "colored":
        tgt, tn = datagen.surface(15000, 31)
        tc = datagen.texture(tgt)
        gt = datagen.gt_transform((-0.4, 0.6, 0.8), (0.004, -0.003, 0.002))
        src, sn, sc = datagen.make_source(tgt, gt, 33, 34, 2e-4, attrs=[(tn, True), (tc, False)])
        return src, sn, sc, tgt, tn, tc
    tgt, tn = datagen.surface(20000, 71)
    tc = datagen.texture(tgt)
    gt = datagen.gt_transform((-0.6, 0.8, 1.2), (0.006, -0.004, 0.005))
    src, sn, sc = datagen.make_source(tgt, gt, 72, 73, 3e-4, attrs=[(tn, True), (datagen.texture(tgt), False)])
    if scene == "cone":
        Rz = np.array([[0, 0, -1], [0, 1, 0], [1, 0, 0]], np.float64)  # e_z -> -e_x
        tgt, tn, src, sn = (np.ascontiguousarray(x.astype(np.float64) @ Rz.T, np.float32) for x in (tgt, tn, src, sn))
    return src, sn, sc, tgt, tn, tc


# the loop replays start at a pose with a large translation, so that an update composed on the wrong side (T U instead of
# U T, off by (R_U - I) t) is far outside the bound; the source is shifted back by it, its normals are unchanged
REPLAY_INIT = np.eye(4, dtype=np.float32)
REPLAY_INIT[:3, 3] = [0.5, -1.0, 2.0]


def _shifted(p):
    return np.ascontiguousarray(p - REPLAY_INIT[:3, 3], np.float32)


def _move(src, sn, scov, T):
    """the source at pose T in float64, rounded once, and the bound on how far the device's float32 copy may be"""
    Rm, t = T[:3, :3].astype(np.float64), T[:3, 3].astype(np.float64)
    P = src.astype(np.float64) @ Rm.T + t
    out = dict(src=P.astype(np.float32))
    if sn is not None:
        out["src_nrm"] = (sn.astype(np.float64) @ Rm.T).astype(np.float32)
    if scov is not None:
        out["src_cov"] = np.einsum("ij,njk,lk->nil", Rm, scov.astype(np.float64), Rm).astype(np.float32)
    scale = (np.abs(src).max() * np.abs(Rm).sum(1).max() + np.abs(t).max())
    return out, 4 * U * scale


def bounded_gradient(n):
    """a colour gradient of bounded size.  The fitted one of this scene has outliers that make the colored 6x6 system
    ill-conditioned (kappa ~ 4e6): the float32 solve's forward-error bound then exceeds the update itself"""
    return (0.3 * datagen.unit_normals(n, 74)).astype(np.float32)


def _setup(kind, lam=0.968, scene=None, plain=False, shift=False):
    src, sn, sc, tgt, tn, tc = loop_scene(scene)
    if shift:
        src = _shifted(src)
    r = 0.03
    a = dict(src_nrm=sn, src_col=sc, tgt_nrm=tn, tgt_col=tc)
    s_pc, t_pc = {"p2p": lambda: (cloud(src), cloud(tgt)), "p2plane": lambda: (cloud(src), cloud(tgt, tn)),
                  "symmetric": lambda: (cloud(src, sn), cloud(tgt, tn)),
                  "colored": lambda: (cloud(src, sn, sc), cloud(tgt, tn, tc, grad=bounded_gradient(len(tgt)))
                                      if not plain else R.initialize_pointcloud_for_colored_icp(cloud(tgt, tn, tc), 2 * r)),
                  "gicp": lambda: (R._with_covariances(cloud(src, sn), 1e-3), R._with_covariances(cloud(tgt, tn), 1e-3))}[kind]()
    if kind == "colored":
        a["tgt_grad"] = t_pc._color_gradient.cpu()
    if kind == "gicp":
        a["src_cov"], a["tgt_cov"] = s_pc._covariances.cpu().reshape(-1, 3, 3), t_pc._covariances.cpu().reshape(-1, 3, 3)
    return src, tgt, r, a, s_pc, t_pc


def _run(kind, s_pc, t_pc, r, k, lam=0.968, plain=None):
    crit = R.ICPConvergenceCriteria(0, 0, k)
    if kind == "colored" and plain is not None:
        return R.registration_colored_icp(plain[0], plain[1], r, REPLAY_INIT, crit, lambda_geometric=lam)
    if kind == "gicp" and plain is not None:
        return R.registration_generalized_icp(plain[0], plain[1], r, REPLAY_INIT,
                                              R.TransformationEstimationForGeneralizedICP(1e-3), crit)
    return R.registration_icp(s_pc, t_pc, r, REPLAY_INIT, estimation(kind, lam), crit)


def _first_update_same_sums(kind, sums, n_src, lam):
    """the float64 update from the device's own step sums at the first pose, only the solver's arithmetic charged ->
    (U, bound, {mutant: U})"""
    if kind == "p2p":
        U64, err = icp64.kabsch_from_sums(sums[:15], int(sums[29]), n_src)
        return U64, err, {}
    k = KINDS[kind]
    S32 = np.concatenate([sums[:27].astype(np.float32), [0]]).astype(np.float64)
    dt = -1.0 if kind == "gicp" else 1e-6
    sv = icp64.solve(k, S32, None, dt)
    assert sv["firm"] and sv["ok"]
    mut = {"no_square": icp64.solve(k, S32, None, dt, mutant="no_square")["T"]} if k == icp64.SYMMETRIC else {}
    return sv["T"], sv["err"], mut


STEP_T = datagen.gt_transform((-0.3, 0.5, 0.6), (0.003, -0.002, 0.002)).astype(np.float32)


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_fused_step_sums(kind):
    src, tgt, r, a, s_pc, t_pc = _setup(kind)
    ctx = R.IcpContext(s_pc, t_pc, r, estimation(kind))
    try:
        sums, ci = ctx.step(STEP_T)
    finally:
        ctx.close()
    moved, err = _move(src, a["src_nrm"], a.get("src_cov"), STEP_T)
    m = ci >= 0
    corr = np.stack([np.nonzero(m)[0], ci[m]], 1).astype(np.int32)
    assert sums[29] == len(corr) and len(corr) > 0.9 * len(src)
    aa = dict(a, **{k: v for k, v in moved.items() if k != "src"})
    if kind == "p2p":
        ks = icp64.kabsch_sums(moved["src"], tgt, corr)
        bound = ks["bound"] + err * np.concatenate([np.full(3, len(corr)), np.zeros(3), np.repeat(np.abs(tgt[corr[:, 1]]).sum(0)[None], 3, 0).reshape(9)])
        _note(kind, "step sums", icp64.sums_ratio(sums[:15], ks["S"], bound))
        return
    keys = {"p2plane": ("tgt_nrm",), "symmetric": ("src_nrm", "tgt_nrm"),
            "colored": ("src_col", "tgt_nrm", "tgt_col", "tgt_grad"), "gicp": ("src_cov", "tgt_cov")}[kind]
    ne = icp64.normal_equations(KINDS[kind], moved["src"], tgt, corr, src_err=err, **{x: aa[x] for x in keys})
    _note(kind, "step sums", icp64.sums_ratio(sums[:28], ne["S"], ne["bound"]))


REPLAY_K = 6


def _replay(kind, lam=0.968, scene=None, plain=False):
    src, tgt, r, a, s_pc, t_pc = _setup(kind, lam, scene, plain, shift=True)
    pl = None
    if plain:
        s0, sn0, sc0, t0, tn0, tc0 = loop_scene(scene)
        s0 = _shifted(s0)
        pl = (cloud(s0, sn0, sc0), cloud(t0, tn0, tc0)) if kind == "colored" else (cloud(s0, sn0), cloud(t0, tn0))
    poses = [_run(kind, s_pc, t_pc, r, k, lam, plain=pl) for k in range(REPLAY_K + 1)]
    ctx = R.IcpContext(s_pc, t_pc, r, estimation(kind, lam))
    skipped = 0
    try:
        for k in range(REPLAY_K):
            Tk = poses[k].transformation
            sums, ci = ctx.step(Tk)
            m = ci >= 0
            corr = np.stack([np.nonzero(m)[0], ci[m]], 1).astype(np.int32)
            # fitness and inlier_rmse of the run capped at k updates, from the step's own search
            n_c = int(sums[29])
            assert poses[k].fitness == np.float32(n_c) / np.float32(len(src))
            moved, err = _move(src, a["src_nrm"], a.get("src_cov"), Tk)
            err = err * (k + 1)  # the loop's working copy took k float32 updates, not one
            rm = np.sqrt(sums[28] / n_c)
            assert abs(poses[k].inlier_rmse - rm) <= err + 8 * U * rm
            T_next = poses[k + 1].transformation.astype(np.float64)
            if k == 0:
                # the run's first update comes from the same opening as step(T_0) (the pristine source moved once by
                # T_0), so its sums are c_0: the update and its composition are held to the solver's own arithmetic,
                # and the same bound rejects the update composed on the right (and Symmetric without R R)
                U0, e0, mut = _first_update_same_sums(kind, sums, len(src), lam)
                T0 = Tk.astype(np.float64)
                want, berr = icp64.compose(U0, T0, e0)
                _note(kind, "first update, own sums", _frac(np.linalg.norm(T_next - want), berr))
                size = np.linalg.norm(U0 - np.eye(4))
                print("%s first update: bound %.3g of the update" % (kind, berr / size))
                assert berr <= 0.1 * size
                ratios = {"right": np.linalg.norm(T_next - icp64.compose(U0, T0, e0, mutant="right")[0]) / berr}
                for name, Um in mut.items():
                    ratios[name] = np.linalg.norm(T_next - icp64.compose(Um, T0, e0)[0]) / berr
                print("%s replay mutants: %s" % (kind, {x: "%.3g" % y for x, y in ratios.items()}))
                assert min(ratios.values()) >= MUTANT_MARGIN
            aa = dict(a, **{x: v for x, v in moved.items() if x != "src"})
            Uk, uerr, firm = _restated(kind, moved["src"], tgt, corr, aa, lam, src_err=err,
                                       det_thresh=-1.0 if kind == "gicp" else 1e-6)
            if not firm:  # the bound cannot decide the gate: only fitness and rmse are checked at this step
                skipped += 1
                continue
            want, berr = icp64.compose(Uk, Tk.astype(np.float64), uerr)
            _note(kind, "loop update", _frac(np.linalg.norm(T_next - want), berr))
    finally:
        ctx.close()
    print("%s replay: %d of %d updates checked against the restated update" % (kind, REPLAY_K - skipped, REPLAY_K))
    # the fitted colour gradient of registration_colored_icp can make the bound unable to decide the gate: most
    # updates must still be checked; every one where the gradient is bounded
    assert skipped == 0 if not plain else skipped <= REPLAY_K // 2
    return poses


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_loop_replay(kind):
    poses = _replay(kind)
    assert poses[-1].fitness > 0.9


def test_loop_replay_colored_lambda():
    """registration_colored_icp with lambda_geometric = 0.5 (its target gradient built inside)"""
    poses = _replay("colored", lam=0.5, scene="colored", plain=True)
    assert poses[-1].fitness > 0.9


def test_loop_replay_generalized_icp_cone():
    """registration_generalized_icp on a scene turned so that part of its normals fall inside the -e1 cone, where the
    covariance is diag(eps, 1, 1) and the first update's rows take FastEigen3x3's diagonal branch"""
    src, sn, sc, tgt, tn, tc = loop_scene("cone")
    assert (tn[:, 0] < -0.99).mean() > 0.005 and (sn[:, 0] < -0.99).mean() > 0.005
    from oracle import oracle_py as orc
    cov_s, cov_t = orc.covariances_from_normals(sn, 1e-3), orc.covariances_from_normals(tn, 1e-3)
    ident = np.stack([np.arange(len(src))] * 2, 1)
    assert icp64.rows(icp64.GICP, src, src, ident, src_cov=cov_s, tgt_cov=cov_s)["diag"].mean() > 0.005
    _replay("gicp", scene="cone", plain=True)


def test_zz_report():
    """the largest observed deviation from icp64, per estimator and check, as a fraction of its bound"""
    for k in sorted(STATS):
        print("ICP64 %-40s %.3g" % (k, STATS[k]))
