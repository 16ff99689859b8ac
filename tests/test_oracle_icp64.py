"""The CPU oracle's ICP estimators (orc.jtj_jtr, orc.solve_jtj, orc.kabsch) against the float64 restatement of
cupoch_b200/testing/icp64.py, within the bounds derived there, for all five estimators: surface pairs at the origin and
10^3 units from it, lambda_geometric in {0, 0.25, 0.968, 1}, GICP normals nearly parallel, axis-aligned and inside the
-e1 cone, 1, 2 and 5 correspondences, rank-deficient systems, and mutants of the restatement that the same bounds must
reject by a wide margin."""
import functools

import numpy as np
import pytest

from cupoch_b200.testing import datagen, icp64

KINDS = {"p2plane": icp64.P2PLANE, "symmetric": icp64.SYMMETRIC, "colored": icp64.COLORED, "gicp": icp64.GICP}
LAMBDAS = [0.0, 0.25, 0.968, 1.0]
MUTANT_MARGIN = 10.0  # a mutant's worst sum or pose must be at least this many bounds away


@functools.lru_cache(None)
def surface_scene(far=0.0, n=4000, seed=11):
    from oracle import oracle_py as orc
    orc.build()
    tgt, tn = datagen.surface(n, seed)
    tc = datagen.texture(tgt)
    gt = datagen.gt_transform((-0.4, 0.6, 0.8), (0.004, -0.003, 0.002))
    src, sn, sc = datagen.make_source(tgt, gt, seed + 1, seed + 2, 3e-4, attrs=[(tn, True), (datagen.texture(tgt), False)])
    if far:
        src, tgt = (src + np.float32(far)).astype(np.float32), (tgt + np.float32(far)).astype(np.float32)
    corr, _, _ = orc.correspondences(src, tgt, 0.05)
    nbr, _, _ = orc.search(tgt, tgt, 30, radius=0.1, kdtree=True)
    grad = orc.color_gradient(tgt, tn, tc, nbr)
    attrs = dict(src_nrm=sn, src_col=sc, src_cov=orc.covariances_from_normals(sn, 1e-3), tgt_nrm=tn, tgt_col=tc,
                 tgt_grad=grad, tgt_cov=orc.covariances_from_normals(tn, 1e-3))
    return src, tgt, corr, attrs


@functools.lru_cache(None)
def normal_scene(case, n=600, seed=5):
    """source = target + a small offset, matched i <-> i, with GICP's edge-case normals"""
    from oracle import oracle_py as orc
    rng = np.random.Generator(np.random.PCG64(seed))
    tgt = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    src = (tgt + rng.normal(0, 2e-3, (n, 3))).astype(np.float32)
    tn = datagen.unit_normals(n, seed + 1)
    if case == "parallel":  # the source normal within 1e-3 .. 0.3 rad of the target's
        th = np.exp(rng.uniform(np.log(1e-3), np.log(0.3), n))[:, None]
        u = np.cross(tn, datagen.unit_normals(n, seed + 2))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        sn = np.cos(th) * tn + np.sin(th) * u
    elif case == "axis":
        tn = np.zeros((n, 3), np.float32)
        tn[np.arange(n), rng.integers(0, 3, n)] = rng.choice([-1.0, 1.0], n)
        sn = tn.copy()
    else:  # "cone": n . e1 < -0.99, where the covariance is diag(eps, 1, 1) whatever the normal
        v = rng.normal(0, 0.08, (n, 3))
        v[:, 0] = -1.0
        tn = v / np.linalg.norm(v, axis=1, keepdims=True)
        sn = np.where((tn[:, :1] < -0.99) & (rng.random((n, 1)) < 0.5), tn, datagen.unit_normals(n, seed + 3))
    tn, sn = tn.astype(np.float32), np.asarray(sn, np.float32)
    corr = np.stack([np.arange(n), np.arange(n)], 1).astype(np.int32)
    attrs = dict(src_cov=orc.covariances_from_normals(sn, 1e-3), tgt_cov=orc.covariances_from_normals(tn, 1e-3))
    return src, tgt, corr, attrs


def _needs(kind, attrs):
    keys = {icp64.P2PLANE: ("tgt_nrm",), icp64.SYMMETRIC: ("src_nrm", "tgt_nrm"),
            icp64.COLORED: ("src_col", "tgt_nrm", "tgt_col", "tgt_grad"), icp64.GICP: ("src_cov", "tgt_cov")}[kind]
    return {k: attrs[k] for k in keys}


def _check_sums(orc, kind, src, tgt, corr, attrs, lam=0.968, label=""):
    a = _needs(kind, attrs)
    got = orc.jtj_jtr(kind, src, tgt, corr, lambda_geometric=lam, **a)
    ne = icp64.normal_equations(kind, src, tgt, corr, lambda_geometric=lam, **a)
    ratio = icp64.sums_ratio(got[:28], ne["S"], ne["bound"])
    print("%s %s lambda %g: %d correspondences, sums max_ratio %.3g" % (label, icp64.NAMES[kind], lam, len(corr), ratio))
    assert ratio <= 1.0, (got[:28] - ne["S"]) / ne["bound"]
    return got, ne


def _check_per_correspondence(orc, kind, src, tgt, corr, attrs, lam=0.968, label="", take=150):
    a = _needs(kind, attrs)
    sel = corr[np.linspace(0, len(corr) - 1, min(take, len(corr))).astype(int)]
    got = np.stack([orc.jtj_jtr(kind, src, tgt, c[None], lambda_geometric=lam, **a)[:28] for c in sel])
    S, B = icp64.per_correspondence(kind, src, tgt, sel, lambda_geometric=lam, **a)
    ratio = icp64.sums_ratio(got, S, B)
    print("%s %s lambda %g: per-correspondence max_ratio %.3g" % (label, icp64.NAMES[kind], lam, ratio))
    assert ratio <= 1.0
    return got, sel, ratio


def _check_solve(orc, kind, got, det_thresh=1e-6, label=""):
    """orc.solve_jtj on the float32 sums against the float64 solve of the same sums"""
    u, b = got[:21].astype(np.float32), got[21:27].astype(np.float32)
    dt = -1.0 if kind == icp64.GICP else det_thresh
    ok, T = orc.solve_jtj(u, b, dt)
    sv = icp64.solve(kind, np.concatenate([u, b, [0]]).astype(np.float64), None, dt)
    if sv["firm"]:
        assert ok == sv["ok"], (sv["det"], dt)
    if kind == icp64.SYMMETRIC and ok:
        R = T[:3, :3].astype(np.float64)
        T = T.copy()
        T[:3, :3] = R @ R
    if ok and sv["ok"]:
        d = np.linalg.norm(T.astype(np.float64) - sv["T"])
        print("%s %s: solve |dT| %.3g, bound %.3g (ratio %.3g), kappa %.3g" % (
            label, icp64.NAMES[kind], d, sv["err"], d / sv["err"], sv["inv_norm"] * np.linalg.norm(icp64.unpack(got)[0], 2)))
        assert d <= sv["err"]
    return ok, T, sv


@pytest.mark.parametrize("far", [0.0, 1000.0])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_surface_sums_and_solve(orc, kind, far):
    src, tgt, corr, attrs = surface_scene(far)
    k = KINDS[kind]
    for lam in (LAMBDAS if k == icp64.COLORED else [0.968]):
        got, ne = _check_sums(orc, k, src, tgt, corr, attrs, lam, "far %g" % far)
        _check_per_correspondence(orc, k, src, tgt, corr, attrs, lam, "far %g" % far)
        ok, T, _ = _check_solve(orc, k, got, label="far %g" % far)
        # and the pose from the restated sums, bound carried through the solve
        sv = icp64.solve(k, ne["S"], ne["bound"], -1.0 if k == icp64.GICP else 1e-6)
        assert ok == sv["ok"] or not sv["firm"]
        if ok:
            d = np.linalg.norm(T.astype(np.float64) - sv["T"])
            print("   pose from restated sums |dT| %.3g bound %.3g" % (d, sv["err"]))
            assert d <= sv["err"]


@pytest.mark.parametrize("case", ["parallel", "axis", "cone"])
def test_gicp_normals(orc, case):
    src, tgt, corr, attrs = normal_scene(case)
    _check_sums(orc, icp64.GICP, src, tgt, corr, attrs, label=case)
    got, sel, _ = _check_per_correspondence(orc, icp64.GICP, src, tgt, corr, attrs, label=case, take=len(corr))
    _check_solve(orc, icp64.GICP, orc.jtj_jtr(icp64.GICP, src, tgt, corr, **attrs), label=case)
    rw = icp64.rows(icp64.GICP, src, tgt, corr, **attrs)
    # the branch each scene is for: the general one for nearly parallel normals (but for the few pairs that both fall
    # in the cone), the diagonal one for axis normals and for the cone pairs
    assert rw["diag"].mean() < 0.05 if case == "parallel" else rw["diag"].mean() > (0.9 if case == "axis" else 0.3)


def test_gicp_diagonal_rows_weigh_500_times_more(orc):
    """the translation block of one GICP correspondence's J^T J is W^2: M^-1 / max coefficient in FastEigen3x3's general
    branch, M^-1 itself when M^-1 is exactly diagonal -- about 500 times more for eps = 1e-3 covariances"""
    # (no zero components in the general-branch normals: an exactly vanishing projection makes the reference's row NaN,
    # which hazard 8 drops)
    n = np.float32([[-1.0, 0.0, 0.0], [-0.995, 0.0, np.sqrt(1 - 0.995 ** 2)], [0.36, 0.48, 0.8], [0.6, 0.48, 0.64]])
    cov = orc.covariances_from_normals(n.astype(np.float32), 1e-3)
    p = np.zeros((4, 3), np.float32)
    tblock = []
    for i in range(4):
        corr = np.array([[i, i]], np.int32)
        got = orc.jtj_jtr(icp64.GICP, p, p, corr, src_cov=cov, tgt_cov=cov)
        S, B = icp64.per_correspondence(icp64.GICP, p, p, corr, src_cov=cov, tgt_cov=cov)
        assert icp64.sums_ratio(got[:28], S[0], B[0]) <= 1.0
        A, _ = icp64.unpack(got)
        tblock.append(np.trace(A[3:, 3:]))
    assert icp64.rows(icp64.GICP, p, p, np.stack([np.arange(4)] * 2, 1), src_cov=cov, tgt_cov=cov)["diag"].tolist() == [
        True, True, False, False]
    # M = 2 (I - (1 - eps) n n^T), M^-1 = (I + (1 / eps - 1) n n^T) / 2 with trace 501 (eps = 1e-3).  Diagonal branch:
    # W^2 = M^-1, trace 501; general branch: W^2 = M^-1 / mc, mc = (1 + 999 max n_i^2) / 2, here 320 and 205
    mc = (1.0 + 999.0 * (n[2:].astype(np.float64) ** 2).max(1)) / 2.0
    np.testing.assert_allclose(tblock[:2], 501.0, rtol=1e-4)
    np.testing.assert_allclose(tblock[2:], 501.0 / mc, rtol=1e-3)
    assert min(tblock[:2]) / max(tblock[2:]) > 200


@pytest.mark.parametrize("count", [1, 2, 5])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_few_correspondences(orc, kind, count):
    """rank <= 5 systems: the sums hold, and the gate refuses every one of them (|det| is rounding noise)"""
    src, tgt, corr, attrs = surface_scene()
    k = KINDS[kind]
    got, _ = _check_sums(orc, k, src, tgt, corr[::997][:count], attrs, label="count %d" % count)
    ok, _, sv = _check_solve(orc, k, got, label="count %d" % count)
    if k != icp64.GICP and count < 5:
        assert sv["firm"] and not sv["ok"] and not ok


def test_rank_deficient_ldlt_zero_pivot(orc):
    """z = 0.5 lattice, normals +e_z, point-to-plane: the columns of rotation about z and of x / y translation are
    exactly zero, LDLT meets exact zero pivots; with the gate off the solve must still return a finite x with
    A64 x = -b64 within the solver's backward error"""
    from cupoch_b200.testing import normals64
    tgt, _ = normals64.lattice_plane("z", side=30, spacing=0.01)
    tn = np.tile(np.float32([[0, 0, 1]]), (len(tgt), 1))
    rng = np.random.Generator(np.random.PCG64(3))
    src = (tgt + rng.normal(0, 1e-3, tgt.shape)).astype(np.float32)
    corr = np.stack([np.arange(len(tgt))] * 2, 1).astype(np.int32)
    got, ne = _check_sums(orc, icp64.P2PLANE, src, tgt, corr, dict(tgt_nrm=tn), label="lattice")
    A, b = icp64.unpack(got[:28].astype(np.float32).astype(np.float64))
    assert (A[:, [2, 3, 4]] == 0).all() and (b[[2, 3, 4]] == 0).all()
    ok, T = orc.solve_jtj(got[:21].astype(np.float32), got[21:27].astype(np.float32), -1.0)
    assert ok and np.isfinite(T).all()
    from scipy.spatial.transform import Rotation
    x = np.concatenate([Rotation.from_matrix(T[:3, :3].astype(np.float64)).as_rotvec(), T[:3, 3].astype(np.float64)])
    nA = np.linalg.norm(A)
    res = np.linalg.norm(A @ x + b)
    bound = nA * (icp64.LDLT_K * icp64.U * np.linalg.norm(x) + icp64.SE3_K * icp64.U * (1 + np.linalg.norm(x))) \
        + icp64.U * np.linalg.norm(b)
    print("zero-pivot solve: |A x + b| %.3g, bound %.3g" % (res, bound))
    assert res <= bound
    # the gate refuses the same system
    assert not orc.solve_jtj(got[:21].astype(np.float32), got[21:27].astype(np.float32), 1e-6)[0]


def test_det_gate_decisions(orc):
    """thresholds a factor 10^3 either side of |det|: the oracle's decision is the float64 one"""
    src, tgt, corr, attrs = surface_scene()
    got = orc.jtj_jtr(icp64.P2PLANE, src, tgt, corr, tgt_nrm=attrs["tgt_nrm"])
    S32 = np.concatenate([got[:27].astype(np.float32), [0]]).astype(np.float64)
    det = abs(icp64.solve(icp64.P2PLANE, S32, None, -1.0)["det"])
    for thr, want in ((det / 1e3, True), (det * 1e3, False)):
        sv = icp64.solve(icp64.P2PLANE, S32, None, thr)
        assert sv["firm"] and sv["ok"] == want
        assert orc.solve_jtj(got[:21].astype(np.float32), got[21:27].astype(np.float32), np.float32(thr))[0] == want


@pytest.mark.parametrize("far", [0.0, 1000.0])
def test_kabsch(orc, far):
    src, tgt, corr, _ = surface_scene(far)
    for n_model in (None, len(corr)):
        T, S = orc.kabsch(src, tgt, corr, n_model)
        ks = icp64.kabsch_sums(src, tgt, corr)
        assert icp64.sums_ratio(S[:15], ks["S"], ks["bound"]) <= 1.0
        T64, err = icp64.kabsch(src, tgt, corr, n_model)
        d = np.linalg.norm(T.astype(np.float64) - T64)
        print("kabsch far %g n_model %s: |dT| %.3g bound %.3g" % (far, n_model, d, err))
        assert d <= err


# ---- mutants: the tolerances above must be able to see a subtle error ----------------------------------------------
def _mutant_ratio(orc, kind, mutant, src, tgt, corr, attrs, lam):
    a = _needs(kind, attrs)
    sel = corr[np.linspace(0, len(corr) - 1, min(150, len(corr))).astype(int)]
    got = np.stack([orc.jtj_jtr(kind, src, tgt, c[None], lambda_geometric=lam, **a)[:28] for c in sel])
    _, B = icp64.per_correspondence(kind, src, tgt, sel, lambda_geometric=lam, **a)
    Sm, _ = icp64.per_correspondence(kind, src, tgt, sel, lambda_geometric=lam, mutant=mutant, **a)
    return icp64.sums_ratio(got, Sm, B)


@pytest.mark.parametrize("kind,mutant,lam,scene", [
    ("colored", "grad_sign", 0.25, "surface"), ("colored", "grad_sign", 0.968, "surface"),
    ("colored", "lambda_swap", 0.25, "surface"), ("colored", "lambda_swap", 0.968, "surface"),
    ("gicp", "minv", 0.968, "surface"), ("gicp", "unscaled", 0.968, "surface"), ("gicp", "minv", 0.968, "cone"),
    ("gicp", "unscaled", 0.968, "parallel")])
def test_row_mutants_rejected(orc, kind, mutant, lam, scene):
    src, tgt, corr, attrs = surface_scene() if scene == "surface" else normal_scene(scene)
    ratio = _mutant_ratio(orc, KINDS[kind], mutant, src, tgt, corr, attrs, lam)
    print("mutant %s / %s lambda %g on %s: rejected at %.3g bounds" % (kind, mutant, lam, scene, ratio))
    assert ratio >= MUTANT_MARGIN


INIT = datagen.gt_transform((1.0, -2.0, 3.0), (0.5, -1.0, 2.0))


def _pulled_back(src, attrs):
    """the source moved by INIT^-1 (float64, rounded once), so that a loop started at INIT meets the target again"""
    Ti = np.linalg.inv(INIT)
    Ri = Ti[:3, :3]
    out = dict(attrs)
    out["src_nrm"] = (attrs["src_nrm"].astype(np.float64) @ Ri.T).astype(np.float32)
    out["src_cov"] = np.einsum("ij,njk,lk->nil", Ri, attrs["src_cov"].astype(np.float64), Ri).astype(np.float32)
    return (src.astype(np.float64) @ Ri.T + Ti[:3, 3]).astype(np.float32), out


@pytest.mark.parametrize("kind", ["p2p"] + sorted(KINDS))
def test_pose_mutants_rejected(orc, kind):
    """one update of the oracle's RegistrationICP loop started at a pose with a large translation: T_1 = U T_0 with U the
    float64 solve of the loop's own sums (only the solver's arithmetic charged).  The same bound rejects the update
    composed on the right (T_0 U) and, for Symmetric, the update without its R R step"""
    src0, tgt, _, attrs0 = surface_scene()
    src, attrs = _pulled_back(src0, attrs0)
    k = icp64.P2P if kind == "p2p" else KINDS[kind]
    r = 0.05
    kw = {} if k == icp64.P2P else _needs(k, attrs)
    res = orc.registration_icp(k, src, tgt, r, init=INIT.astype(np.float32), relative_fitness=0, relative_rmse=0,
                               max_iteration=1, **kw)
    # the loop's first update, from the source as the loop moved it (float32, by INIT) and its own correspondences
    T0 = INIT.astype(np.float32)
    moved = orc.transform_points(src, T0)
    corr, _, _ = orc.correspondences(moved, tgt, r)
    if k == icp64.P2P:
        _, S = orc.kabsch(moved, tgt, corr, len(src))
        U64, err = icp64.kabsch_from_sums(S[:15], len(corr), len(src))
        mut = {}
    else:
        mv = dict(kw)
        if "src_nrm" in mv:
            mv["src_nrm"] = orc.transform_normals(mv["src_nrm"], T0)
        if "src_cov" in mv:
            mv["src_cov"] = orc.rotate_covariances(mv["src_cov"], T0)
        got = orc.jtj_jtr(k, moved, tgt, corr, **mv)
        S32 = np.concatenate([got[:27].astype(np.float32), [0]]).astype(np.float64)
        dt = -1.0 if k == icp64.GICP else 1e-6
        sv = icp64.solve(k, S32, None, dt)
        assert sv["firm"] and sv["ok"]
        U64, err = sv["T"], sv["err"]
        mut = {"no_square": icp64.solve(k, S32, None, dt, mutant="no_square")["T"]} if k == icp64.SYMMETRIC else {}
    T1 = res["transformation"].astype(np.float64)
    want, berr = icp64.compose(U64, T0.astype(np.float64), err)
    d = np.linalg.norm(T1 - want)
    print("%s: oracle loop's first update |dT| %.3g, bound %.3g (%.3g of the update's size)" % (
        kind, d, berr, berr / np.linalg.norm(U64 - np.eye(4))))
    assert d <= berr
    assert berr <= 0.1 * np.linalg.norm(U64 - np.eye(4))  # the bound is far below the update it checks
    ratios = {"right": np.linalg.norm(T1 - icp64.compose(U64, T0.astype(np.float64), err, mutant="right")[0]) / berr}
    for name, Um in mut.items():
        ratios[name] = np.linalg.norm(T1 - icp64.compose(Um, T0.astype(np.float64), err)[0]) / berr
    print("pose mutants %s: %s" % (kind, {a: "%.3g" % b for a, b in ratios.items()}))
    assert min(ratios.values()) >= MUTANT_MARGIN


def test_kabsch_model_size_mutant_rejected(orc):
    """Kabsch's centroids and H are divided by the model size, not the correspondence count (kabsch.cu:76,107): with
    half the source matched, dividing by the count lands far outside the bound"""
    src, tgt, corr, _ = surface_scene()
    half = corr[::2]
    T, _ = orc.kabsch(src, tgt, half, len(src))
    T64, err = icp64.kabsch(src, tgt, half, len(src))
    Tm, _ = icp64.kabsch(src, tgt, half, len(half))
    assert np.linalg.norm(T.astype(np.float64) - T64) <= err
    ratio = np.linalg.norm(T.astype(np.float64) - Tm) / err
    print("mutant p2p / count instead of model size: rejected at %.3g bounds" % ratio)
    assert ratio >= MUTANT_MARGIN
