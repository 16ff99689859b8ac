"""Float64 restatement of ComputeSHOTFeature (registration/shot.cu:63-255) in plain numpy, one point at a time and
vectorised over its neighbours.  Used by tests/ to check the CPU oracle against an independent computation.

It takes float32 inputs and the neighbour lists as arguments (idx[n, k] int32 with -1 for empty slots, d2[n, k]
float32), so the search is not part of what it checks.  It keeps the reference's quirks:
  - the frame: w = radius - sqrt(d2) (negative beyond radius), cov = sum w q q^T / sum w over the listed points other
    than the point itself (by index); z / x are the eigenvectors of the smallest / largest eigenvalue, each flipped when
    fewer than half of q.axis are >= 0; y = z x x.  Fewer than 5 such points -> an all-zero row;
  - cos_desc = clip(z . n_i, -1, 1) with the point's OWN normal; bindist = 5 (1 + cos_desc); step = round half up,
    so cos_desc = 1 gives column 10;
  - a neighbour at distance 0 adds nothing; frame coordinates below 1e-30 in magnitude are 0; the sector bits, the
    shell, inclination and azimuth interpolation as the reference writes them; the row is divided by its norm if > 0.

The oracle and the device compute in float32 (and FastEigen3x3 instead of an iterative eigen-solver), so a point whose
computation passes close to a decision -- a sign test, the step rounding, a branch threshold, a frame-sign vote, or
nearly equal eigenvalues -- can differ by more than rounding.  shot64 returns each point's smallest relative distance to
such a decision (its margin); points with a margin above a small slack must agree to rounding.
"""
import numpy as np

DIM = 352
N_BINS = 10
MIN_NB = 5
SECTORS = 32
RAD_45, RAD_90, RAD_135, RAD_PI_7_8 = np.pi / 4, np.pi / 2, 3 * np.pi / 4, 7 * np.pi / 8


def _frame(q, w):
    """-> (x, y, z, margin): the local reference frame and its smallest relative decision distance"""
    cov = (w[:, None, None] * q[:, :, None] * q[:, None, :]).sum(0) / w.sum()
    ev, V = np.linalg.eigh(cov)  # ascending
    scale = max(abs(ev).max(), 1e-300)
    gap = min(ev[1] - ev[0], ev[2] - ev[1]) / scale
    # FastEigen3x3 returns the eigenvalues of cov / (its largest coefficient) unscaled, and the reference picks the min /
    # max of those: a negative largest coefficient (weights beyond the radius) swaps the two axes
    mc = cov.max()
    lo, hi = (2, 0) if mc < 0 else (0, 2)
    z, x = V[:, lo].copy(), V[:, hi].copy()
    qn = np.linalg.norm(q, axis=1)
    qn[qn == 0] = 1.0
    # a relative eigen-gap g turns the float32 solver's axes by ~1e-7 / g: counted as a margin of g / 100
    margin = min(gap / 100, abs(mc) / max(abs(cov).max(), 1e-300))
    for axis in (x, z):
        s = q @ axis
        pos = int((s >= 0).sum())
        if pos < len(q) - pos:
            axis *= -1.0
        vote = abs(2 * pos - len(q))  # a tie keeps the solver's arbitrary sign
        margin = min(margin, 0.0 if vote == 0 else 1.0, np.min(np.abs(s) / qn))
    return x, np.cross(z, x), z, margin


def shot_point(p, nrm, i, idx, d2, radius):
    """-> (row [352] float64, margin) of point i"""
    ft = np.zeros(DIM)
    keep = (idx >= 0) & (idx != i)
    j, dd = idx[keep], d2[keep].astype(np.float64)
    if len(j) < MIN_NB:
        return ft, np.inf
    q = p[j] - p[i]
    x_ax, y_ax, z_ax, margin = _frame(q, radius - np.sqrt(dd))
    cos_desc = np.clip(z_ax @ nrm[i], -1.0, 1.0)
    bindist = (1.0 + cos_desc) * N_BINS / 2.0
    step = int(np.floor(bindist + 0.5))
    frac = bindist - step
    margin = min(margin, abs(abs(frac) - 0.5))  # the step rounding (frac = 0 is continuous)
    r12, r34, r14 = radius / 2, radius * 3 / 4, radius / 4
    for qq, d in zip(q, np.sqrt(dd)):
        if d == 0:
            continue
        x, y, z = qq @ x_ax, qq @ y_ax, qq @ z_ax
        x, y, z = (0.0 if abs(v) < 1e-30 else v for v in (x, y, z))
        bit4 = 1 if (y > 0 or (y == 0 and x < 0)) else 0
        bit3 = (1 - bit4) if (x > 0 or (x == 0 and y > 0)) else bit4
        desc = ((bit4 << 3) + (bit3 << 2)) << 1
        if x * y > 0 or x == 0:
            desc += 0 if abs(x) >= abs(y) else 4
        else:
            desc += 4 if abs(x) > abs(y) else 0
        desc += 1 if z > 0 else 0
        desc += 2 if d > r12 else 0
        vol = desc * (N_BINS + 1)
        iw = 1.0 - abs(frac)
        if frac > 0:
            ft[vol + (step + 1) % N_BINS] += frac
        else:
            ft[vol + (step - 1 + N_BINS) % N_BINS] += -frac
        if d > r12:
            rd = (d - r34) / r12
            if d > r34:
                iw += 1 - rd
            else:
                iw += 1 + rd
                ft[(desc - 2) * (N_BINS + 1) + step] -= rd
        else:
            rd = (d - r14) / r12
            if d < r14:
                iw += 1 + rd
            else:
                iw += 1 - rd
                ft[(desc + 2) * (N_BINS + 1) + step] += rd
        inc = np.arccos(np.clip(z / d, -1.0, 1.0))
        if inc > RAD_90 or (inc == RAD_90 and z <= 0):
            idist = (inc - RAD_135) / RAD_90
            if inc > RAD_135:
                iw += 1 - idist
            else:
                iw += 1 + idist
                ft[(desc + 1) * (N_BINS + 1) + step] -= idist
        else:
            idist = (inc - RAD_45) / RAD_90
            if inc < RAD_45:
                iw += 1 + idist
            else:
                iw += 1 - idist
                ft[(desc - 1) * (N_BINS + 1) + step] += idist
        if y != 0 or x != 0:
            az = np.arctan2(y, x)
            sel = desc >> 2
            ad = (az - (-RAD_PI_7_8 + RAD_45 * sel)) / RAD_45
            ad = max(-0.5, min(ad, 0.5))
            if ad > 0:
                iw += 1 - ad
                ft[((desc + 4) % SECTORS) * (N_BINS + 1) + step] += ad
            else:
                iw += 1 + ad
                ft[((desc - 4 + SECTORS) % SECTORS) * (N_BINS + 1) + step] -= ad
        ft[vol + step] += iw
        # the discontinuous decisions: the sector bits, the outer shell, the upper / lower half (the interpolations at
        # r / 4, 3 r / 4, 45, 135 degrees and at the sector centres are continuous)
        margin = min(margin, abs(x) / d, abs(y) / d, abs(z) / d, abs(abs(x) - abs(y)) / d, abs(d - r12) / radius,
                     abs(inc - RAD_90))
    norm = np.sqrt((ft * ft).sum())
    if norm > 0:
        ft /= norm
    return ft, margin


def shot64(pts, nrm, idx, d2, radius):
    """-> (rows [n, 352] float64, margin [n] float64; +inf for rows that are zero by the neighbour count)"""
    p = np.asarray(pts, np.float32).astype(np.float64)
    nv = np.asarray(nrm, np.float32).astype(np.float64)
    n = len(p)
    rows, margins = np.zeros((n, DIM)), np.full(n, np.inf)
    for i in range(n):
        rows[i], margins[i] = shot_point(p, nv, i, idx[i], d2[i], float(radius))
    return rows, margins
