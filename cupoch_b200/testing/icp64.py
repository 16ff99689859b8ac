"""Float64 restatement of the five ICP estimators over an explicit correspondence list: rows, normal equations, the
6x6 solve with its determinant gate, the pose update and ComputeRMSE, each with an error bound derived below.  Used by
tests/ to check the CPU oracle and the device kernels against a computation that shares neither their code nor their
float32 arithmetic.

Inputs are float32 arrays (points [n, 3], normals, colours, colour gradients [n, 3], covariances [n, 3, 3]) and the
correspondence list corr[m, 2] = (source index, target index), so the search is not part of what is checked.  Every
value is converted to float64 once and nothing is rounded to float32 afterwards.

Rows (J[q, 6], r[q]) of one correspondence (vs, vt the matched points, d = vs - vt):
  Point-to-plane   transformation_estimation.cu:34-56   J = (vs x nt, nt), r = d . nt
  Symmetric        transformation_estimation.cu:58-90   nn = ns + nt: J = ((vs + vt) x nn, nn), r = d . nn
  Colored          colored_icp.cu:150-216               two rows, sg = sqrt(lambda), sp = sqrt(1 - lambda):
                     J0 = sg (vs x nt, nt), r0 = sg d . nt;
                     vs' = vs - (d . nt) nt (projection onto the tangent plane), I(c) = (r + g + b) / 3,
                     gm = -gt^T (I - nt nt^T), J1 = sp (vs x gm, gm), r1 = sp (I(cs) - (gt . (vs' - vt) + I(ct)))
  GICP             generalized_icp.cu:63-105            three rows i: J_i = w_i^T (-[vs]x, I), r_i = w_i . d, w_i the
                   rows of W = SqrtMatrix3x3((Ct + Cs)^-1) (eigenvalue.inl:93-178), which is NOT the square root of
                   M^-1 = (Ct + Cs)^-1:
                     * general branch: FastEigen3x3 divides by the signed largest coefficient mc of M^-1 and never
                       scales the eigenvalues back, so W = sqrt(M^-1 / mc) (DESIGN parity hazard 6);
                     * M^-1 exactly diagonal (its off-diagonal squares sum to 0, eigenvalue.inl:106): the raw diagonal
                       is returned, W = sqrt(M^-1), about sqrt(mc) ~ 22 times larger for GICP's eps = 1e-3 covariances
                       (M^-1 ~ diag(500, 0.5, 0.5)).  Both covariances are exactly diagonal for axis-aligned normals
                       and for every normal with n_x < -0.99, whose covariance skips the rotation (generalized_icp.cu:
                       18-36); such rows weigh ~500 times more in the sums.  Reference-faithful, restated as such.
                   A row with a non-finite entry is dropped (DESIGN parity hazard 8).
  Point-to-point   kabsch.cu:42-120: sums of vs, vt and vs vt^T (the device's step layout).

Normal equations (utility/eigen.inl:118-145): the 21 upper-triangle sums of J_a J_b (row-major a <= b), the 6 sums of
J_a r, sum r^2; `mag` holds the matching sums of |J_a J_b|, |J_a r|, r^2.

Solve (utility/eigen.cu:75-122): x = -A^-1 b, T = exp(x) with t = x[3:] (eigen.cu:28-50); the determinant gate
|det A| < det_thresh refuses the step (identity) except for GICP, which has no gate (generalized_icp.cu:176-179).
Symmetric squares R and keeps t (transformation_estimation.cu:315-346).  The loop composes on the left, T <- U T
(registration.cu:159).  Kabsch divides the centroids and H by the model size, not the correspondence count
(kabsch.cu:76,107).

ComputeRMSE: P2P sqrt(mean |d|^2) (transformation_estimation.cu:109-134); P2Plane sqrt(mean r^2), 0 without target
normals (:144-192); Symmetric sqrt(mean (r^2)^2) (:224-286, the squared error squared again, hazard 7); GICP
sqrt(mean d^T W d), W as above (generalized_icp.cu:134-151); Colored the plain sum of r0^2 + r1^2 (colored_icp.cu:
303-327, hazard 7).

The bounds.  U = 2^-23.
  Row entries.  Each float32 entry is a short chain of roundings over float32 inputs, so its error is at most ROW_K U
  times the sum of the magnitudes of the terms it is formed from (|vs| |nt| for a cross product: this is what grows
  for points far from the origin; |d| |nt| for a residual; |gt| (|vs| + |vt|) for the photometric residual, whose
  projection fma(-dn, nt, vs) rounds at the scale of vs).  A source known only to within src_err (the loop's working
  copy is transformed in float32 once per update) adds src_err times each entry's derivative in vs.
  GICP's W.  W^T W = W^2 is all the sums depend on (J^T J = P^T W^2 P with P = (-[vs]x, I), J^T r = P^T W^2 d), so
  its bound is one on W^2, E = GICP_C U (kappa(M) lam2 + min(p^2 / g, p / sqrt(U)) + ROW_K lam2) per correspondence,
  lam the eigenvalues of the matrix FastEigen3x3 sees (M^-1 / mc), g its smallest eigenvalue gap, p = sqrt(sum (lam_i -
  mean)^2 / 6) the scale FastEigen3x3 divides by:
    kappa(M) lam2   the float32 inverse by cofactors loses kappa(M) ulps;
    p^2 / g         FastEigen3x3 takes the eigenvalues q + 2 p cos(angle) from angle = acos(h) / 3, h = det(B) / 2p^3;
                    an error of a few U in h moves angle by U / sqrt(1 - h^2) ~ U p / g and the eigenvalues by
                    U p^2 / g (normals64.py's term, with p <= lam2 in place of lam2); at g -> 0 acos(1 - d) =
                    sqrt(2 d) makes it saturate at p sqrt(2 U).  Nearly parallel normals (the usual case for matched points) meet
                    exactly there: M^-1 ~ diag(500, 0.5, 0.5) has two nearly equal small eigenvalues.
  Sums.  |dS_ab| <= sum over rows of (|J_a| e_b + e_a |J_b| + e_a e_b), plus for GICP E c_a c_b with c the column
  absolute sums of P (||d||_1 for the residual), plus the float64 summation's m 2^-52 mag.
  Pose.  With dA, db the Frobenius norms of the sums' bounds plus their rounding to float32 and LDLT's backward error
  (LDLT_K U ||A||), the forward error of the solve is |dx| <= 2 ||A^-1|| (dA |x| + db) (kappa(A) times the relative
  perturbation, first order, the 2 covering the second-order term while ||A^-1|| dA <= 1/2).  exp moves R by at most
  sqrt(2) |dw| and t by |dt|; its float32 evaluation adds SE3_K U per entry; R R doubles the rotation's error; the
  composition U T multiplies it by ||T||.
  Determinant gate.  |d det / det| <= ||A^-1||_2 dA 6; a decision is firm when |det| and det_thresh lie further apart
  than that (both ways), and only firm decisions are checked.
Constants are fixed once below.  ROW_K, LDLT_K and SE3_K follow from operation counts; GICP_C is empirical (its comment
says how it was set), because FastEigen3x3's acos error has no closed-form constant here."""
import numpy as np

U = 2.0 ** -23
P2P, P2PLANE, SYMMETRIC, COLORED, GICP = 1, 2, 3, 4, 5
NAMES = {P2P: "p2p", P2PLANE: "p2plane", SYMMETRIC: "symmetric", COLORED: "colored", GICP: "gicp"}
# rounding steps in one row entry: the longest chain (the photometric residual: intensity sum and division, the
# projection fma, subtraction, dot3's three roundings, the addition of I(ct), the subtraction from I(cs), the product
# with sp) has 9; every entry is charged 16 so that a term this derivation misses by a factor of two still fits
ROW_K = 16.0
# GICP's W^2, empirical: the largest ratio of observed error to the bound at GICP_C = 1, over every GICP input of
# tests/test_oracle_icp64.py (printed as max_ratio, which is measured at GICP_C = 4), is below 1.4; 4 leaves a margin
# near three
GICP_C = 4.0
# LDLT of a 6x6 SPD matrix: Higham (Accuracy and Stability, thm 10.5) |dA| <= gamma_{n+1} |L||D||L^T|, and
# || |L||D||L^T| || <= n ||A|| for a symmetric positive semidefinite A: (n + 1) n = 42
LDLT_K = 42.0
# se(3) exp and the 4x4 product: float32 cos / sin rounded from double and at most four roundings per entry of R
SE3_K = 8.0
CHUNK = 1 << 17  # correspondences per vectorised pass


def _f64(a, cols=3):
    return None if a is None else np.asarray(a, np.float32).reshape(-1, cols).astype(np.float64)


def _cross_mag(a, b):
    """|a| x |b| as the magnitudes each cross-product entry is formed from"""
    a, b = np.abs(a), np.abs(b)
    return np.stack([a[:, 1] * b[:, 2] + a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] + a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] + a[:, 1] * b[:, 0]], 1)


def intensity(c):
    return c.sum(1) / 3.0


# ---- GICP's W ------------------------------------------------------------------------------------------------------
def gicp_w(Cs, Ct, mode="reference"):
    """W per correspondence (and the data of its bound).  mode: "reference" (the two branches above), or the mutants
    "minv" (M^-1 in place of W) and "unscaled" (sqrt(M^-1): no max-coefficient scaling in the general branch)
    -> W[m, 3, 3], lam[m, 3] (of the matrix FastEigen3x3 sees), kappa(M)[m], diagonal-branch mask[m]"""
    M = Cs + Ct
    Mi = np.linalg.inv(M)
    off = Mi[:, [0, 0, 1], [1, 2, 2]]
    diag = (off == 0).all(1)
    mc = Mi.reshape(-1, 9).max(1)
    A = np.where((diag | (mode == "unscaled"))[:, None, None], Mi, Mi / mc[:, None, None])
    lam, V = np.linalg.eigh(A)
    lam_c = np.maximum(lam, 0.0)
    W = np.einsum("nij,nj,nkj->nik", V, np.sqrt(lam_c), V)
    if mode == "minv":
        W = Mi
    lm = np.linalg.eigvalsh(M)
    kappa = lm[:, 2] / np.maximum(lm[:, 0], 1e-300)
    return W, lam, kappa, diag


# ---- rows ----------------------------------------------------------------------------------------------------------
def rows(kind, src, tgt, corr, src_nrm=None, src_col=None, src_cov=None, tgt_nrm=None, tgt_col=None, tgt_grad=None,
         tgt_cov=None, lambda_geometric=0.968, src_err=0.0, mutant=None):
    """-> dict J [m, q, 6], r [m, q], eJ, er (entry bounds), and for GICP W, E (W^2 bound), P (3 x 6 per row),
    d, diag.  mutant: None or one of "grad_sign", "lambda_swap" (Colored), "minv", "unscaled" (GICP)"""
    corr = np.asarray(corr, np.int64).reshape(-1, 2)
    i, j = corr[:, 0], corr[:, 1]
    vs, vt = _f64(src)[i], _f64(tgt)[j]
    m = len(corr)
    d = vs - vt
    ad = np.abs(d)
    if kind == P2PLANE:
        nt = _f64(tgt_nrm)[j]
        J = np.concatenate([np.cross(vs, nt), nt], 1)[:, None]
        r = (d * nt).sum(1)[:, None]
        eJ = np.concatenate([ROW_K * U * _cross_mag(vs, nt) + src_err * (np.abs(nt).sum(1, keepdims=True) - np.abs(nt)),
                             np.zeros((m, 3))], 1)[:, None]
        er = (ROW_K * U * (ad * np.abs(nt)).sum(1) + src_err * np.abs(nt).sum(1))[:, None]
        return dict(J=J, r=r, eJ=eJ, er=er)
    if kind == SYMMETRIC:
        nt, ns = _f64(tgt_nrm)[j], _f64(src_nrm)[i]
        nn = ns + nt
        sm = vs + vt
        an = np.abs(nn)
        J = np.concatenate([np.cross(sm, nn), nn], 1)[:, None]
        r = (d * nn).sum(1)[:, None]
        # nn and sm are each rounded once; the source normal carries src_err too (rotated with the points)
        eJ = np.concatenate([ROW_K * U * _cross_mag(sm, an) + src_err * (_cross_mag(np.ones_like(sm), an)
                                                                                      + _cross_mag(sm, np.ones_like(an))),
                             ROW_K * U * an + src_err], 1)[:, None]
        er = (ROW_K * U * (ad * an).sum(1) + src_err * (an.sum(1) + ad.sum(1)))[:, None]
        return dict(J=J, r=r, eJ=eJ, er=er)
    if kind == COLORED:
        nt, gt = _f64(tgt_nrm)[j], _f64(tgt_grad)[j]
        cs, ct = _f64(src_col)[i], _f64(tgt_col)[j]
        lam = float(np.float32(lambda_geometric))
        sg, sp = np.sqrt(lam), np.sqrt(1.0 - lam)
        if mutant == "lambda_swap":
            sg, sp = sp, sg
        if mutant == "grad_sign":
            gt = -gt
        dn = (d * nt).sum(1)
        J0 = sg * np.concatenate([np.cross(vs, nt), nt], 1)
        r0 = sg * dn
        vproj = vs - dn[:, None] * nt
        Is, It = intensity(cs), intensity(ct)
        is0 = (gt * (vproj - vt)).sum(1) + It
        Mt = np.eye(3)[None] - nt[:, :, None] * nt[:, None, :]
        gm = -np.einsum("na,nab->nb", gt, Mt)
        J1 = sp * np.concatenate([np.cross(vs, gm), gm], 1)
        r1 = sp * (Is - is0)
        J = np.stack([J0, J1], 1)
        r = np.stack([r0, r1], 1)
        an, ag = np.abs(nt), np.abs(gt)
        sn1 = an.sum(1, keepdims=True)
        eJ0 = sg * np.concatenate([ROW_K * U * _cross_mag(vs, nt) + src_err * (sn1 - an), ROW_K * U * an], 1)
        egm = ROW_K * U * 2.0 * ag.sum(1, keepdims=True) * np.ones((1, 3))
        agm = np.abs(gm)
        eJ1 = sp * np.concatenate([ROW_K * U * _cross_mag(vs, gm) + _cross_mag(vs, egm)
                                   + src_err * (agm.sum(1, keepdims=True) - agm), egm], 1)
        er0 = sg * (ROW_K * U * (ad * an).sum(1) + src_err * an.sum(1))
        scale = np.abs(vs).max(1) + np.abs(vt).max(1) + np.abs(dn)
        er1 = sp * (ROW_K * U * (Is + It + np.abs(is0) + (ag * np.abs(vproj - vt)).sum(1) + ag.sum(1) * scale)
                    + src_err * agm.sum(1))
        return dict(J=J, r=r, eJ=np.stack([eJ0, eJ1], 1), er=np.stack([er0, er1], 1))
    if kind == GICP:
        Cs = np.asarray(src_cov, np.float32).reshape(-1, 3, 3).astype(np.float64)[i]
        Ct = np.asarray(tgt_cov, np.float32).reshape(-1, 3, 3).astype(np.float64)[j]
        W, lam, kappa, diag = gicp_w(Cs, Ct, {"minv": "minv", "unscaled": "unscaled"}.get(mutant, "reference"))
        P = np.zeros((m, 3, 6))
        P[:, 0, 1], P[:, 0, 2] = vs[:, 2], -vs[:, 1]     # -[vs]x
        P[:, 1, 0], P[:, 1, 2] = -vs[:, 2], vs[:, 0]
        P[:, 2, 0], P[:, 2, 1] = vs[:, 1], -vs[:, 0]
        P[:, :, 3:] = np.eye(3)
        J = np.einsum("nik,nka->nia", W, P)
        r = np.einsum("nik,nk->ni", W, d)
        aW = np.abs(W)
        eJ = np.concatenate([ROW_K * U * np.einsum("nik,nka->nia", aW, np.abs(P[:, :, :3]))
                             + src_err * (aW.sum(2, keepdims=True) - aW), np.zeros((m, 3, 3))], 2)
        er = ROW_K * U * np.einsum("nik,nk->ni", aW, ad) + src_err * aW.sum(2)
        lam2 = np.abs(lam).max(1)
        g = np.min(np.diff(lam, axis=1), 1)
        pp = np.sqrt(((lam - lam.mean(1, keepdims=True)) ** 2).sum(1) / 6.0)  # FastEigen3x3's p
        with np.errstate(divide="ignore", invalid="ignore"):
            eig = np.where(diag, 0.0, np.minimum(pp * pp / g, pp / np.sqrt(U)))
        E = GICP_C * U * (kappa * lam2 + eig + ROW_K * lam2)
        return dict(J=J, r=r, eJ=eJ, er=er, W=W, E=E, P=P, d=d, diag=diag, lam=lam)
    raise ValueError("kind %r" % kind)


# ---- normal equations ----------------------------------------------------------------------------------------------
IU = np.triu_indices(6)


def _ne_chunk(rw):
    J, r, eJ, er = rw["J"], rw["r"], rw["eJ"], rw["er"]
    finite = np.isfinite(J).all(2) & np.isfinite(r)
    J, r = np.where(finite[:, :, None], J, 0.0), np.where(finite, r, 0.0)
    eJ, er = np.where(finite[:, :, None], eJ, 0.0), np.where(finite, er, 0.0)
    Z = np.concatenate([J, r[:, :, None]], 2)           # [m, q, 7]
    E = np.concatenate([eJ, er[:, :, None]], 2)
    aZ = np.abs(Z)
    S = np.einsum("nqa,nqb->ab", Z, Z)
    mag = np.einsum("nqa,nqb->ab", aZ, aZ)
    B = np.einsum("nqa,nqb->ab", aZ, E)
    B = B + B.T + np.einsum("nqa,nqb->ab", E, E)
    if "E" in rw:  # GICP: the W^2 term, E c_a c_b (c = column absolute sums of P, ||d||_1 for the residual)
        c = np.concatenate([np.abs(rw["P"]).sum(1), np.abs(rw["d"]).sum(1, keepdims=True)], 1)
        ok = finite.all(1)
        B = B + np.einsum("n,na,nb->ab", np.where(ok, rw["E"], 0.0), c, c)
    return S, mag, B, int(finite.all(1).sum())


def _pack(M):
    """7x7 (J, r) Gram -> 28 sums in the layout of the sums the library returns"""
    return np.concatenate([M[:6, :6][IU], M[:6, 6], [M[6, 6]]])


def per_correspondence(kind, src, tgt, corr, lambda_geometric=0.968, mutant=None, **attrs):
    """the 28 sums of each correspondence alone -> (S[m, 28], bound[m, 28]): no sum of many rows to hide a wrong row in"""
    rw = rows(kind, src, tgt, corr, lambda_geometric=lambda_geometric, mutant=mutant, **attrs)
    finite = (np.isfinite(rw["J"]).all(2) & np.isfinite(rw["r"]))[:, :, None]
    Z = np.where(finite, np.concatenate([rw["J"], rw["r"][:, :, None]], 2), 0.0)
    E = np.where(finite, np.concatenate([rw["eJ"], rw["er"][:, :, None]], 2), 0.0)
    aZ = np.abs(Z)
    S = np.einsum("nqa,nqb->nab", Z, Z)
    B = np.einsum("nqa,nqb->nab", aZ, E)
    B = B + B.transpose(0, 2, 1) + np.einsum("nqa,nqb->nab", E, E)
    if "E" in rw:
        c = np.concatenate([np.abs(rw["P"]).sum(1), np.abs(rw["d"]).sum(1, keepdims=True)], 1)
        B = B + np.where(finite.all(1)[:, 0], rw["E"], 0.0)[:, None, None] * c[:, :, None] * c[:, None, :]
    pack = (lambda M: np.concatenate([M[:, :6, :6][:, IU[0], IU[1]], M[:, :6, 6], M[:, 6, 6:7]], 1))
    return pack(S), pack(B) + 2.0 ** -52 * np.abs(pack(S))


def normal_equations(kind, src, tgt, corr, lambda_geometric=0.968, src_err=0.0, mutant=None, **attrs):
    """-> dict S[28], mag[28], bound[28] (float64), rows_kept"""
    corr = np.asarray(corr, np.int32).reshape(-1, 2)
    S, mag, B, kept = np.zeros((7, 7)), np.zeros((7, 7)), np.zeros((7, 7)), 0
    for s in range(0, len(corr), CHUNK):
        rw = rows(kind, src, tgt, corr[s:s + CHUNK], lambda_geometric=lambda_geometric, src_err=src_err,
                  mutant=mutant, **attrs)
        a, b, c, k = _ne_chunk(rw)
        S, mag, B, kept = S + a, mag + b, B + c, kept + k
    B = B + len(corr) * 2.0 ** -52 * mag
    return dict(S=_pack(S), mag=_pack(mag), bound=_pack(B), rows_kept=kept)


def kabsch_sums(src, tgt, corr):
    """-> dict S[15] (sum vs, sum vt, sum vs_a vt_b row-major), bound[15] (summation order only: exact products)"""
    corr = np.asarray(corr, np.int64).reshape(-1, 2)
    vs, vt = _f64(src)[corr[:, 0]], _f64(tgt)[corr[:, 1]]
    S = np.concatenate([vs.sum(0), vt.sum(0), np.einsum("na,nb->ab", vs, vt).reshape(9)])
    mag = np.concatenate([np.abs(vs).sum(0), np.abs(vt).sum(0), np.einsum("na,nb->ab", np.abs(vs), np.abs(vt)).reshape(9)])
    return dict(S=S, mag=mag, bound=len(corr) * 2.0 ** -52 * mag)


# ---- solve and pose ------------------------------------------------------------------------------------------------
def unpack(S):
    A = np.zeros((6, 6))
    A[IU] = S[:21]
    A = A + np.triu(A, 1).T
    return A, np.asarray(S[21:27], np.float64)


def se3_exp(x):
    """eigen.cu:28-50 in float64"""
    T = np.eye(4)
    T[:3, 3] = x[3:]
    th = np.linalg.norm(x[:3])
    if th == 0:
        return T
    w = x[:3] / th
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    T[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)
    return T


def solve(kind, S, bound=None, det_thresh=1e-6, mutant=None):
    """-> dict T (4x4 float64 update), ok (step taken), firm (the gate's decision is beyond its margin), det, margin,
    err (Frobenius bound on T), x, dA, db, inv_norm.  bound None: S are the float32 sums the solver itself was given,
    so only its own arithmetic is charged.  mutant "no_square": symmetric without the R R step"""
    S = np.asarray(S, np.float64)
    A, b = unpack(S)
    Ab, bb = unpack(np.zeros(28) if bound is None else bound)
    nA = np.linalg.norm(A)
    dA = np.linalg.norm(Ab) + U * nA + LDLT_K * U * nA
    db = np.linalg.norm(bb) + U * np.linalg.norm(b)
    with np.errstate(all="ignore"):
        det = float(np.linalg.det(A))
        sv = np.linalg.svd(A, compute_uv=False)
        inv_norm = 1.0 / sv[-1] if sv[-1] > 0 else np.inf
        margin = 6.0 * inv_norm * dA * abs(det)
    gate = kind != GICP and det_thresh > 0
    ok = True
    firm = True
    if gate:
        ok = abs(det) >= det_thresh
        firm = (abs(abs(det) - det_thresh) > margin) and np.isfinite(margin)
    out = dict(ok=ok, firm=firm, det=det, margin=margin, dA=dA, db=db, inv_norm=inv_norm)
    if not ok:
        out.update(T=np.eye(4), err=0.0, x=np.zeros(6))
        return out
    x = -np.linalg.lstsq(A, b, rcond=None)[0] if not np.isfinite(inv_norm) else -np.linalg.solve(A, b)
    dx = 2.0 * inv_norm * (dA * np.linalg.norm(x) + db)
    T = se3_exp(x)
    err = np.sqrt(2.0) * dx + dx + 16 * SE3_K * U
    if kind == SYMMETRIC and mutant != "no_square":
        T[:3, :3] = T[:3, :3] @ T[:3, :3]
        err = 2.0 * err
    out.update(T=T, err=err, x=x)
    return out


def compose(Uk, Tk, err_u, mutant=None):
    """the loop's T <- U T (registration.cu:159) -> (T, Frobenius bound); mutant "right": T U"""
    T = Tk @ Uk if mutant == "right" else Uk @ Tk
    return T, err_u * np.linalg.norm(Tk, 2) + 4 * SE3_K * U * np.linalg.norm(Uk) * np.linalg.norm(Tk)


def kabsch(src, tgt, corr, n_model=None, src_err=0.0):
    """kabsch.cu:42-120 in float64 with its divide-by-model-size quirk -> (T, Frobenius bound); src_err as in rows()"""
    corr = np.asarray(corr, np.int64).reshape(-1, 2)
    S = kabsch_sums(src, tgt, corr)["S"]
    n = len(src) if n_model is None else int(n_model)
    extra = src_err * (np.abs(S[3:6]) + len(corr) * np.abs(S[3:6]) / n + np.abs(_f64(tgt)[corr[:, 1]]).sum(0))[None, :] / n
    T, err = kabsch_from_sums(S, len(corr), n, extra)
    return T, err + 2 * src_err


def kabsch_from_sums(S, count, n_model, dH_extra=0.0):
    """the update from the sums (kabsch_sums layout, count correspondences, centroids and H divided by the model size
    n_model) -> (T, Frobenius bound charging the arithmetic after the sums, plus dH_extra on H)"""
    S = np.asarray(S, np.float64)
    n, C = float(n_model), float(count)
    mc, tc = S[0:3] / n, S[3:6] / n
    Sst = S[6:15].reshape(3, 3)
    H = (Sst - np.outer(mc, S[3:6]) - np.outer(S[0:3], tc) + C * np.outer(mc, tc)) / n
    # the float32 centroids and the float32 division of each H entry: the cancellation is at the scale of the terms
    dH = ROW_K * U * (np.abs(Sst) + np.abs(np.outer(mc, S[3:6])) + np.abs(np.outer(S[0:3], tc))
                      + C * np.abs(np.outer(mc, tc))) / n + U * np.abs(H) + dH_extra
    Uu, s, Vt = np.linalg.svd(H)
    V = Vt.T
    dd = np.linalg.det(Uu @ Vt)
    R = V @ np.diag([1.0, 1.0, np.sign(dd) if dd != 0 else 1.0]) @ Uu.T
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = tc - R @ mc
    with np.errstate(divide="ignore"):
        dR = 2.0 * np.linalg.norm(dH) / (s[1] + s[2]) + SE3_K * U
    err = dR + dR * np.linalg.norm(mc) + ROW_K * U * (np.linalg.norm(tc) + np.linalg.norm(mc))
    return T, err


# ---- ComputeRMSE ---------------------------------------------------------------------------------------------------
def rmse(kind, src, tgt, corr, lambda_geometric=0.968, **attrs):
    """-> (value, bound) with the reference's per-kind formula and quirks (module docstring)"""
    corr = np.asarray(corr, np.int64).reshape(-1, 2)
    n = len(corr)
    if n == 0:
        return 0.0, 0.0
    if kind == P2P:
        vs, vt = _f64(src)[corr[:, 0]], _f64(tgt)[corr[:, 1]]
        d2 = ((vs - vt) ** 2).sum(1)
        s, e = d2.sum(), (ROW_K * U * d2).sum()
    else:
        rw = rows(kind, src, tgt, corr, lambda_geometric=lambda_geometric, **attrs)
        r, er = rw["r"], rw["er"]
        if kind == GICP:
            # d^T W d: W itself, whose error is the W^2 bound over 2 sqrt(lam_min) (the derivative of the square root)
            d = rw["d"]
            t = (d * r).sum(1)
            lmin = np.maximum(np.abs(rw["lam"]).min(1), 1e-300)
            eW = rw["E"] / (2.0 * np.sqrt(lmin))
            te = (np.abs(d) * er).sum(1) + eW * np.abs(d).sum(1) ** 2
            ok = np.isfinite(t)
            s, e = t[ok].sum(), te[ok].sum()
        else:
            ok = np.isfinite(r).all(1)
            r, er = r[ok], er[ok]
            t = (r * r).sum(1)
            te = (2 * np.abs(r) * er + er * er).sum(1)
            if kind == SYMMETRIC:
                te = 2 * t * te + te * te
                t = t * t
            s, e = t.sum(), te.sum()
    e = e + n * 2.0 ** -52 * abs(s) + U * abs(s)  # the float32 sum's rounding to float once
    if kind == COLORED:
        return float(s), float(e + U * abs(s))
    v = np.sqrt(max(s, 0.0) / n)
    with np.errstate(divide="ignore", invalid="ignore"):
        ev = min(e / n / (2 * v), np.sqrt(e / n)) if v > 0 else np.sqrt(e / n)
    return float(v), float(ev + 4 * U * v)


def sums_ratio(got, ref, bound):
    """largest |got - ref| / bound over the sums (0 / 0 counts as 0)"""
    got, ref, bound = (np.asarray(a, np.float64) for a in (got, ref, bound))
    diff = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(diff == 0, 0.0, diff / bound)
    return float(np.max(q)) if q.size else 0.0
