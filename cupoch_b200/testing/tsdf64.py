"""Float64 restatements of UniformTSDFVolume's ExtractPointCloud (integration/uniform_tsdfvolume.cu:36-156) and Raycast
(uniform_tsdfvolume.cu:447-639) in plain numpy.  Used by tests/ to check the CPU oracle and the device against an
independent computation.

They take the volume's float32 planes as they are (tw [N, 2] (tsdf, weight), col [planes, N], voxel idx = x res^2 +
y res + z) and the float32 scalars of the volume (voxel length = float32(length) / float32(res)), and compute
everything after that in float64.  The project's deliberate deviations from the reference are restated as the oracle
documents them:
  - ExtractPointCloud emits one row per crossing (sized by its crossings, not by the band voxels), in (x, y, z, axis)
    order;
  - Raycast enters on the box of the cells the march may sample, [-(res/2) vl, (res - 1 - res/2) vl]^3 relative to the
    origin, not on the reference's [0, length]^3; a direction component that is exactly 0 keeps its slab when the
    camera lies inside it and misses otherwise;
  - the march length is len0 + vl + i * (trunc / 2), computed without accumulation; the oracle's rule that a step which
    no longer advances the float32 length ends the march as a miss has no float64 counterpart and is not restated.

Decision margins.  Where float32 can reach a different discrete outcome than float64, the row's result may differ by
more than rounding.  Each row carries the smallest distance (in voxel units) of its float64 computation to such a
threshold:
  - Raycast: the floor of every march sample's grid coordinate (which voxel is read), the entry test len < tmax, the
    bound tests loc in [1, res - 1) and loc -+ 1 in [1, res - 1), |len - lim| at every step, and the (int) of the colour
    voxel.  A march sample's floor only counts where it matters: the voxel on the other side of the integer (or a
    skipped step, when that voxel lies outside the sampled cells) would carry a tsdf of another sign, or the sample is
    one of the two whose values the hit interpolates;
  - ExtractPointCloud: its crossings are decided on the stored float32 values, so only an f0 * f1 that underflows in
    float32 (|f0 f1| < 2^-126) or a normal whose float32 squared norm could underflow can differ; such rows get
    margin 0, every other row an infinite one.
The floors inside GetTSDFAt and InterpolateTrilinearly are not decisions: the trilinear interpolant is continuous, so
either neighbouring base gives the same value up to rounding.  Their distances are returned as `floors` for the record.

Raycast also returns `drift`, a bound (length units) on how far the float32 march length can be from the float64 one
at the row's last step: the entry time's rounding (relative 2^-22 of the slab time, divided by the direction component
that set it) plus half an ulp of the length per accumulated step.
"""
from collections import namedtuple

import numpy as np

EPS32 = 2.0 ** -24  # the unit roundoff of float32
FLT_MIN = 2.0 ** -126

Points64 = namedtuple("Points64", "rows points normals colors margin floors nscale")
Ray64 = namedtuple("Ray64", "hit points normals colors margin drift ts nscale voxel")


def _geometry(length, res, origin):
    vl = float(np.float32(length) / np.float32(res))
    return vl, res // 2, np.asarray(origin, np.float32).astype(np.float64).reshape(3)


class _Field:
    """tsdf lookup by global voxel index over a block [k0, k0 + S)^3 of a res^3 volume (the whole volume by default);
    voxels outside the block read as tsdf 0"""

    def __init__(self, tw, col, res, block):
        self.res = res
        self.k0, self.S = (0, res) if block is None else (int(block[0]), int(block[1]))
        self.f = np.asarray(tw, np.float32)[:, 0].astype(np.float64)
        self.col = None if col is None else np.asarray(col, np.float32).astype(np.float64)

    def local(self, k):
        k = np.asarray(k) - self.k0
        inside = np.all((k >= 0) & (k < self.S), axis=-1)
        kc = np.clip(k, 0, self.S - 1)
        return (kc[..., 0] * self.S + kc[..., 1]) * self.S + kc[..., 2], inside

    def tsdf(self, k):
        i, inside = self.local(k)
        return np.where(inside, self.f[i], 0.0)

    def color(self, k, ct):
        i, _ = self.local(k)
        if ct == 1:
            return self.col[:, i].T / 255.0
        if ct == 2:
            return np.repeat(self.col[0, i][:, None], 3, 1)
        return np.zeros(i.shape + (3,))


def _frac_dist(g):
    return np.abs(g - np.round(g))


def _tsdf_at(F, p, vl):
    """GetTSDFAt (UT:36-65) at rows p [m, 3] (grid-corner coordinates, length units) -> (value, floor distances)"""
    g = p / vl - 0.5
    b = np.floor(g).astype(np.int64)
    r = g - b
    acc = np.zeros(len(p))
    for k in range(8):
        dd = np.array([(k >> 2) & 1, (k >> 1) & 1, k & 1])
        wgt = np.prod(np.where(dd == 1, r, 1 - r), axis=1)
        acc += wgt * F.tsdf(b + dd)
    return acc, _frac_dist(g).min(1)


def extract_point_cloud64(tw, col, length, res, origin, ct, block=None):
    """ExtractPointCloud in float64.  block = (k0, S): tw / col hold only the S^3 voxels from (k0, k0, k0) of a res^3
    volume (the voxels outside read as weight 0); the interior and axis rules use the global indices.
    -> Points64: rows [m, 4] (x, y, z, axis) of every crossing in the oracle's order, points, normals, colours (None
    for NoColor), margin, floors (smallest GetTSDFAt floor distance), nscale (|unnormalised normal|)."""
    vl, h, o = _geometry(length, res, origin)
    F = _Field(tw, col, res, block)
    S, k0 = F.S, F.k0
    f32 = np.asarray(tw, np.float32)[:, 0].reshape(S, S, S)
    w32 = np.asarray(tw, np.float32)[:, 1].reshape(S, S, S)
    band = (w32 != 0) & (f32 < np.float32(0.98)) & (f32 >= np.float32(-0.98))
    g = np.arange(S) + k0
    inner = (g >= 1) & (g <= res - 2)
    interior = inner[:, None, None] & inner[None, :, None] & inner[None, None, :] & band
    f = f32.astype(np.float64)
    mask = np.zeros((S, S, S, 3), bool)
    under = np.zeros((S, S, S, 3), bool)
    for a in range(3):
        sl0 = [slice(None)] * 3
        sl1 = [slice(None)] * 3
        sl0[a], sl1[a] = slice(0, S - 1), slice(1, S)
        ok = np.zeros((S, S, S), bool)
        prod = f[tuple(sl0)] * f[tuple(sl1)]
        ok[tuple(sl0)] = interior[tuple(sl0)] & band[tuple(sl1)] & (prod < 0)
        ax_ok = (g + 1 < res - 1).reshape([-1 if i == a else 1 for i in range(3)])
        mask[..., a] = ok & ax_ok
        und = np.zeros((S, S, S), bool)
        und[tuple(sl0)] = np.abs(prod) < FLT_MIN
        under[..., a] = und
    rows = np.argwhere(mask)
    if len(rows) == 0:
        z = np.zeros((0, 3))
        return Points64(np.zeros((0, 4), np.int64), z, z, None if ct == 0 else z, np.zeros(0), np.zeros(0), np.zeros(0))
    kl, ax = rows[:, :3], rows[:, 3]
    k = kl + k0
    f0 = f[kl[:, 0], kl[:, 1], kl[:, 2]]
    k1 = k + np.eye(3, dtype=np.int64)[ax]
    f1 = F.tsdf(k1)
    r0, r1 = np.abs(f0), np.abs(f1)
    p = (k + 0.5) * vl
    pi = p[np.arange(len(p)), ax]
    p[np.arange(len(p)), ax] = (pi * r1 + (pi + vl) * r0) / (r0 + r1)
    points = p + o - h * vl
    hg = float(0.99 * np.float64(np.float32(vl)))
    n = np.zeros_like(p)
    floors = np.full(len(p), np.inf)
    for a in range(3):
        e = np.zeros(3)
        e[a] = hg
        v1, d1 = _tsdf_at(F, p + e, vl)
        v0, d0 = _tsdf_at(F, p - e, vl)
        n[:, a] = v1 - v0
        floors = np.minimum(floors, np.minimum(d0, d1))
    nscale = np.linalg.norm(n, axis=1)
    normals = np.where(nscale[:, None] > 0, n / np.where(nscale > 0, nscale, 1)[:, None], n)
    colors = None
    if ct != 0:
        c0, c1 = F.color(k, ct), F.color(k1, ct)
        colors = (c0 * r1[:, None] + c1 * r0[:, None]) / (r0 + r1)[:, None]
    # the float32 squared norm of a normal this small can underflow (Eigen then leaves it unnormalised)
    margin = np.where(under[kl[:, 0], kl[:, 1], kl[:, 2], ax] | (nscale < 1e-18), 0.0, np.inf)
    return Points64(np.concatenate([k, ax[:, None]], 1), points, normals, colors, margin, floors, nscale)


def _interp(F, p):
    """InterpolateTrilinearly (UT:447-484) at rows p [m, 3] in grid units (p >= 0.5 on every axis)"""
    b = np.floor(p - 0.5).astype(np.int64)
    a = p - (b + 0.5)
    acc = np.zeros(len(p))
    for k in range(8):
        dd = np.array([(k >> 2) & 1, (k >> 1) & 1, k & 1])
        acc += F.tsdf(b + dd) * np.prod(np.where(dd == 1, a, 1 - a), axis=1)
    return acc


def camera_rays64(K, E, w, h):
    """per pixel (row-major): the unit ray direction and the camera centre of the world-to-camera E, in float64 from
    the float32 K and E: dir = R^T ((x - cx) / fx, (y - cy) / fy, 1) / norm, centre = -R^T t"""
    K = np.asarray(K, np.float32).astype(np.float64)
    E = np.asarray(E, np.float32).astype(np.float64).reshape(4, 4)
    R, tt = E[:3, :3], E[:3, 3]
    ys, xs = np.divmod(np.arange(w * h), w)
    q = np.stack([(xs - K[0, 2]) / K[0, 0], (ys - K[1, 2]) / K[1, 1], np.ones(w * h)], 1)
    d = q @ R
    dn = np.linalg.norm(d, axis=1)
    return d / np.where(dn > 0, dn, 1)[:, None], -R.T @ tt, dn


def raycast64(tw, col, length, res, origin, ct, K, E, trunc, w, h, block=None):
    """Raycast in float64 for a w x h image.  block as for extract_point_cloud64 (voxels outside read as tsdf 0).
    -> Ray64 with one row per pixel: hit (bool), points, normals, colours (NaN rows for misses; zeros for NoColor),
    margin (voxel units), drift (length units), ts (the hit's ray length), nscale (|unnormalised normal|), voxel (the
    colour voxel's indices, -1 for misses)."""
    vl, hh, o = _geometry(length, res, origin)
    F = _Field(tw, col, res, block)
    trunc = float(np.float32(trunc))
    step = trunc * 0.5
    L = res * vl
    lo, hi = -hh * vl, (res - 1 - hh) * vl
    d, c, dn = camera_rays64(K, E, w, h)
    m = w * h
    t = np.broadcast_to(c - o, (m, 3)).copy()
    ok = dn > 0
    margin = np.full(m, np.inf)
    tmin, tmax = np.full(m, -np.inf), np.full(m, np.inf)
    err_in, err_out = np.zeros(m), np.zeros(m)
    for a in range(3):
        z = d[:, a] == 0
        ok &= ~z | ((t[:, a] >= lo) & (t[:, a] <= hi))
        margin = np.where(z, np.minimum(margin, np.minimum(np.abs(t[:, a] - lo), np.abs(t[:, a] - hi)) / vl), margin)
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.where(d[:, a] > 0, lo - t[:, a], hi - t[:, a]) / d[:, a]
            x = np.where(d[:, a] > 0, hi - t[:, a], lo - t[:, a]) / d[:, a]
            # the float32 slab time: the direction component carries ~4 eps absolute, the division 1 eps relative
            err = lambda T: np.abs(T) * (4 * EPS32 / np.abs(d[:, a]) + 2 * EPS32) + 2 * EPS32 * (np.abs(t[:, a]) + abs(lo) + abs(hi)) / np.abs(d[:, a])  # noqa: E731
            ein, eout = err(e), err(x)
        upd_in, upd_out = ~z & (e > tmin), ~z & (x < tmax)
        tmin, err_in = np.where(upd_in, e, tmin), np.where(upd_in, ein, err_in)
        tmax, err_out = np.where(upd_out, x, tmax), np.where(upd_out, eout, err_out)
    err_in = np.where(tmin > 0, err_in, 0.0)  # max(tmin, 0) = 0 exactly for a camera inside the box
    len0 = np.maximum(tmin, 0.0)
    margin = np.where(ok, np.minimum(margin, np.abs(len0 - tmax) / vl), margin)
    ok &= len0 < tmax
    len0 = np.where(ok, len0 + vl, 0.0)
    lim = len0 + L * np.sqrt(2.0)
    # the initial cell: [0, res - 1) per axis, else a miss
    gi = (t + d * len0[:, None]) / vl
    ki = np.floor(gi).astype(np.int64) + hh
    ok &= np.all((ki >= 0) & (ki < res - 1), axis=1)
    f = np.where(ok, F.tsdf(np.clip(ki, 0, res - 1)), 0.0)
    dist_prev = _frac_dist(gi).min(1)  # floor distance of the sample whose value f is
    # the initial floor matters when the voxel across the integer would be outside [0, res - 1) or of another sign
    for a in range(3):
        side = np.where(gi[:, a] - np.floor(gi[:, a]) < 0.5, -1, 1)
        alt = ki.copy()
        alt[:, a] += side
        alt_out = (alt[:, a] < 0) | (alt[:, a] >= res - 1)
        fa = F.tsdf(np.clip(alt, 0, res - 1))
        matters = alt_out | (np.sign(fa) != np.sign(f))
        margin = np.where(ok & matters, np.minimum(margin, _frac_dist(gi[:, a])), margin)
    hit = np.zeros(m, bool)
    active = ok.copy()
    nsteps = np.zeros(m)
    ts_hit = np.full(m, np.nan)
    pts, nrm, cols = (np.full((m, 3), np.nan) for _ in range(3))
    nscale = np.full(m, np.nan)
    voxel = np.full((m, 3), -1, np.int64)
    i = 0
    while active.any():
        ln = len0 + i * step
        near = active & (np.abs(ln - lim) / vl < margin)
        margin = np.where(near, np.abs(ln - lim) / vl, margin)
        active &= ln < lim
        if not active.any():
            break
        nsteps = np.where(active, i + 1, nsteps)
        idx = np.nonzero(active)[0]
        s = ln[idx] + step
        g = (t[idx] + d[idx] * s[:, None]) / vl
        k = np.floor(g).astype(np.int64) + hh
        inr = np.all((k >= 1) & (k < res - 1), axis=1)
        fnew = np.where(inr, F.tsdf(np.clip(k, 0, res - 1)), f[idx])
        fp = f[idx]
        # a floor that picks between voxels of different signs (or between a read and a skip that would change the
        # sign of the carried value) is a decision
        for a in range(3):
            side = np.where(g[:, a] - np.floor(g[:, a]) < 0.5, -1, 1)
            alt = k.copy()
            alt[:, a] += side
            alt_in = np.all((alt >= 1) & (alt < res - 1), axis=1)
            fa = np.where(alt_in, F.tsdf(np.clip(alt, 0, res - 1)), fp)
            matters = np.sign(fa) != np.sign(fnew)
            dd = _frac_dist(g[:, a])
            margin[idx] = np.where(matters, np.minimum(margin[idx], dd), margin[idx])
        dist_now = _frac_dist(g).min(1)
        stop_miss = inr & (fp < 0) & (fnew > 0)
        is_hit = inr & (fp > 0) & (fnew < 0)
        f[idx] = fnew
        if is_hit.any():
            hj = idx[is_hit]
            margin[hj] = np.minimum(margin[hj], np.minimum(dist_now[is_hit], dist_prev[hj]))
            a_, b_ = fp[is_hit], fnew[is_hit]
            ts = ln[hj] - (step * a_) / (b_ - a_)
            vx = t[hj] + d[hj] * ts[:, None]
            loc = vx / vl + hh
            bound = np.minimum(np.abs(loc - 1), np.abs(loc - (res - 1)))
            bound = np.minimum(bound, np.minimum(np.abs(loc + 1 - (res - 1)), np.abs(loc - 1 - 1)))
            margin[hj] = np.minimum(margin[hj], bound.min(1))
            good = np.all((loc >= 1) & (loc < res - 1) & (loc + 1 < res - 1) & (loc - 1 >= 1), axis=1)
            n = np.zeros((len(hj), 3))
            for a in range(3):
                e = np.zeros(3)
                e[a] = 1.0
                sp, sm = np.clip(loc + e, 0.5, res - 1), np.clip(loc - e, 0.5, res - 1)
                n[:, a] = _interp(F, sp) - _interp(F, sm)
            nn = np.linalg.norm(n, axis=1)
            good &= nn > 0
            margin[hj] = np.minimum(margin[hj], _frac_dist(loc).min(1))  # the colour voxel's (int)
            gh = hj[good]
            hit[gh] = True
            ts_hit[gh] = ts[good]
            pts[gh] = vx[good] + o
            nrm[gh] = n[good] / nn[good][:, None]
            nscale[gh] = nn[good]
            vk = np.floor(loc[good]).astype(np.int64)
            voxel[gh] = vk
            cols[gh] = F.color(vk, ct)
        dist_prev[idx] = np.where(inr, dist_now, dist_prev[idx])
        active[idx[stop_miss | is_hit]] = False
        i += 1
    lmax = np.where(ok, len0 + nsteps * step, 0.0)
    drift = err_in + (nsteps + 2) * EPS32 * np.abs(lmax) + 2 * EPS32 * np.abs(len0)
    return Ray64(hit, pts, nrm, cols, margin, drift, ts_hit, nscale, voxel)
