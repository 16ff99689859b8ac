"""Float64 restatement of EstimateNormals (estimate_normals.cu:38-127) over given neighbour lists, and the analytic
GICP covariance that covariances_from_normals (generalized_icp.cu:18-61) approximates.  Used by tests/ to check the CPU
oracle and the device kernels against an independent computation.

Like features64.py it takes float32 points and the neighbour lists idx[n, k] (int32, -1 for empty slots) as
arguments, so the search is not part of what it checks: give it the lists the library's own search returns
(orc.search on the CPU, KDTreeFlann on the device).  Lattices have exact distance ties that only that search's tie
rule settles.

Normals
  - fewer than 3 listed neighbours (k = 0 included): exactly (0, 0, 1);
  - otherwise the centred float64 covariance sum (p - m)(p - m)^T / cnt, m the float64 mean, and a batched
    np.linalg.eigh: eigenvalues lam0 <= lam1 <= lam2, eigenvectors v0, v1, v2.  The normal is v0 up to sign;
  - a covariance that is exactly zero (every neighbour is the same point): exactly (1, 0, 0), the first column of the
    identity FastEigen3x3 returns for a zero matrix (eigenvalue.inl:98-104);
  - always: finite, unit length within UNIT_TOL.

The bound (check_normals).  The kernel's covariance differs from the float64 one by E, with
    |E| <= C err,   err = 2^-23 lam2 + cnt 2^-53 |m|^2:
the first term is the rounding of each coefficient to float32; the second is the float64 cancellation of
E[xx^T] - E[x]E[x]^T, a sum of cnt terms of size |m|^2 (|m| = the neighbourhood's distance from the origin).  By
Davis-Kahan that moves an eigenvector by C err / gap.  FastEigen3x3 adds its own error: it takes the eigenvalues from
acos of a value that tends to +-1 as two eigenvalues meet, so they carry an error of about 2^-23 lam2^2 / gap, and the
eigenvector it derives from them one of 2^-23 (lam2 / gap)^2.  The computed normal n must therefore satisfy
    sin angle(n, v0) <= C (err + 2^-23 lam2^2 / g0) / g0,  g0 = lam1 - lam0  (planes, curved surfaces)
    |n . v2|         <= C (err + 2^-23 lam2^2 / g2) / g2,  g2 = lam2 - lam1  (also lines, where lam0 == lam1 and
                                                                          any n perpendicular to v2 is right)
Both are checked at every point; where a gap vanishes its bound exceeds 1 and the check holds trivially, so an
isotropic neighbourhood is only held to the finite-and-unit rule.  C = NORMAL_C, measured (see its comment).

GICP covariances
  For a unit normal n the reference's R diag(eps, 1, 1) R^T, R the rotation taking e1 to n, is I - (1 - eps) n n^T.
  Its Rodrigues form divides by 1 + n_x and is skipped below n_x = -0.99: there R = I and the result is
  diag(eps, 1, 1) whatever the normal (gicp_cov64 returns that mask)."""
import numpy as np

U = 2.0 ** -23
# Measured on every input of tests/test_oracle_normals64.py and tests/test_gpu_normals64.py: the largest ratio of
# sin angle(n, v0) or |n . v2| to its bound at C = 1 (printed as max_ratio) is below 0.9; 2 leaves a margin of two.
NORMAL_C = 2.0
UNIT_TOL = 4 * U       # | |n| - 1 |: a few roundings of the normalisation
ROW_CHUNK = 1 << 18    # rows per vectorised pass (bounds the [rows, k, 3] temporaries)


def pca64(pts, idx):
    """-> dict of float64 arrays: cnt[n], lam[n, 3] ascending, V[n, 3, 3] (column j = eigenvector of lam[:, j]),
    mean2[n] = |m|^2, zero[n] (covariance exactly 0, cnt >= 3)"""
    P = np.asarray(pts, np.float32).reshape(-1, 3).astype(np.float64)
    idx = np.asarray(idx, np.int32)
    n, k = idx.shape
    cnt = (idx >= 0).sum(1)
    cov = np.zeros((n, 3, 3))
    mean = np.zeros((n, 3))
    for s in range(0, n, ROW_CHUNK):
        I = idx[s:s + ROW_CHUNK]
        use = (I >= 0)[:, :, None]
        Q = np.where(use, P[np.maximum(I, 0)], 0.0)
        c = np.maximum(cnt[s:s + ROW_CHUNK], 1)[:, None]
        m = Q.sum(1) / c
        D = np.where(use, Q - m[:, None, :], 0.0)
        cov[s:s + ROW_CHUNK] = np.einsum("nki,nkj->nij", D, D) / c[:, :, None]
        mean[s:s + ROW_CHUNK] = m
    lam, V = np.linalg.eigh(cov)
    zero = (cnt >= 3) & (cov == 0).all((1, 2))
    return dict(cnt=cnt, lam=lam, V=V, mean2=(mean * mean).sum(1), zero=zero)


def check_normals(nrm, pts, idx, label="", C=NORMAL_C):
    """assert the module's rules for the normals nrm[n, 3] computed from (pts, idx); -> dict of counts and the largest
    measured ratio (printed)"""
    nrm = np.asarray(nrm, np.float32).reshape(-1, 3)
    r = pca64(pts, idx)
    cnt, lam, V = r["cnt"], r["lam"], r["V"]
    few = cnt < 3
    bad = few & ~(nrm == np.float32([0, 0, 1])).all(1)
    assert not bad.any(), "%s: %d points with < 3 neighbours are not (0, 0, 1); first %d: %r" % (
        label, int(bad.sum()), int(np.argmax(bad)), nrm[np.argmax(bad)])
    zero = r["zero"]
    bad = zero & ~(nrm == np.float32([1, 0, 0])).all(1)
    assert not bad.any(), "%s: %d zero covariances are not (1, 0, 0); first %d: %r" % (
        label, int(bad.sum()), int(np.argmax(bad)), nrm[np.argmax(bad)])
    n64 = nrm.astype(np.float64)
    assert np.isfinite(n64).all(), "%s: %d non-finite normals" % (label, int((~np.isfinite(n64)).any(1).sum()))
    norm = np.linalg.norm(n64, axis=1)
    bad = np.abs(norm - 1) > UNIT_TOL
    assert not bad.any(), "%s: %d normals not of unit length; first %d: |n| = %r" % (
        label, int(bad.sum()), int(np.argmax(bad)), norm[np.argmax(bad)])
    gen = ~few & ~zero
    nh = n64 / norm[:, None]
    err = U * lam[:, 2] + cnt * 2.0 ** -53 * r["mean2"]
    sin0 = np.linalg.norm(np.cross(nh, V[:, :, 0]), axis=1)
    dot2 = np.abs((nh * V[:, :, 2]).sum(1))
    # a point passes a check when sin / |dot| is within the bound, or when the bound is at least 1 (neither exceeds 1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        g0, g2 = lam[:, 1] - lam[:, 0], lam[:, 2] - lam[:, 1]
        b0 = (err + U * lam[:, 2] ** 2 / g0) / g0
        b2 = (err + U * lam[:, 2] ** 2 / g2) / g2
        ratio0 = np.where(gen, sin0 / b0, 0.0)
        ratio2 = np.where(gen, dot2 / b2, 0.0)
        b0, b2 = C * b0, C * b2
    fail0 = gen & (sin0 > b0) & ~(b0 >= 1)
    fail2 = gen & (dot2 > b2) & ~(b2 >= 1)
    held0 = gen & (b0 < 1)
    held2 = gen & (b2 < 1)
    info = dict(points=len(nrm), few=int(few.sum()), zero=int(zero.sum()), plane_checked=int(held0.sum()),
                line_checked=int(held2.sum()), free=int((gen & ~held0 & ~held2).sum()),
                max_ratio=float(max(ratio0[held0].max(initial=0.0), ratio2[held2].max(initial=0.0))))
    print("%s normals: %s" % (label, info))
    fail = fail0 | fail2
    if fail.any():
        i = int(np.argmax(fail))
        deg = np.degrees(np.arcsin(np.minimum(sin0, 1.0)))
        raise AssertionError(
            "%s: %d of %d normals outside the bound (%d more than 1 degree off v0); point %d: n %r, v0 %r, lam %r, "
            "|m|^2 %.6g, sin(n, v0) %.3g (bound %.3g), |n.v2| %.3g (bound %.3g)"
            % (label, int(fail.sum()), len(nrm), int((fail & (deg > 1)).sum()), i, nrm[i], V[i, :, 0], lam[i],
               r["mean2"][i], sin0[i], b0[i], dot2[i], b2[i]))
    return info


# ---- clouds at the solver's edges ----------------------------------------------------------------------------------
def lattice_plane(plane, side=60, spacing=0.01, c=0.5, seed=0):
    """side x side lattice with the given spacing on an axis plane "x", "y" or "z" (= c), on "xy" (x = y), or on a
    plane of random orientation through (c, c, c) ("random"); rows shuffled.  -> (points, unit normal[3])"""
    rng = np.random.Generator(np.random.PCG64(seed))
    g = np.arange(side) * spacing
    a, b = (m.ravel() for m in np.meshgrid(g, g, indexing="ij"))
    if plane in ("x", "y", "z"):
        ax = "xyz".index(plane)
        p = np.zeros((len(a), 3))
        p[:, ax] = c
        p[:, [i for i in range(3) if i != ax]] = np.stack([a, b], 1)
        nrm = np.eye(3)[ax]
    elif plane == "xy":
        p = np.stack([a, a, b], 1)
        nrm = np.array([1.0, -1.0, 0.0]) / np.sqrt(2.0)
    else:
        R = np.linalg.qr(rng.standard_normal((3, 3)))[0]
        p = np.stack([a, b, np.zeros_like(a)], 1) @ R.T + c
        nrm = R[:, 2]
    return np.ascontiguousarray(p[rng.permutation(len(p))], np.float32), nrm


def line(n, direction, spacing=0.01, seed=0):
    """n points every `spacing` along a line through (0.5, 0.5, 0.5), rows shuffled"""
    rng = np.random.Generator(np.random.PCG64(seed))
    d = np.asarray(direction, np.float64)
    d /= np.linalg.norm(d)
    p = 0.5 + (rng.permutation(n) * spacing)[:, None] * d
    return p.astype(np.float32)


def cube_lattice(side, spacing=0.125):
    """side^3 lattice (exact coordinates): every inner point's 7 or 27 nearest form an isotropic neighbourhood"""
    g = np.arange(side) * spacing
    return np.stack([m.ravel() for m in np.meshgrid(g, g, g, indexing="ij")], 1).astype(np.float32)


def duplicated(p, times=4, seed=0):
    """every point `times` times, rows shuffled"""
    rng = np.random.Generator(np.random.PCG64(seed))
    q = np.repeat(np.asarray(p, np.float32), times, 0)
    return np.ascontiguousarray(q[rng.permutation(len(q))])


def gicp_cov64(nrm, eps):
    """-> (analytic I - (1 - eps) n n^T [n, 3, 3] in float64, mask of the rows the reference's c < -0.99 branch takes)"""
    N = np.asarray(nrm, np.float32).reshape(-1, 3).astype(np.float64)
    A = np.eye(3) - (1.0 - float(np.float32(eps))) * N[:, :, None] * N[:, None, :]
    return A, np.asarray(nrm, np.float32).reshape(-1, 3)[:, 0] < np.float32(-0.99)
