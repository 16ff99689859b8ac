"""Float64 model of OccupancyGrid::Insert (occupancygrid.cu:462-526), SetFreeArea and the point queries, in plain numpy.
Used by tests/ to check the CPU oracle and the device against the geometry they are meant to compute, not against a
restatement of the same ray walk.

Inputs.  The model takes the float32 start and end points the library forms, and nothing of its algorithm after that:
start = viewpoint - origin and end = ranged - origin, both rounded to float32, where ranged is the point itself for a hit
and viewpoint + (d / |d|) max_range (float32, that operand order) for a ray cut at max_range (`form_rays`).  Whether a
ray is cut is decided on the float32 distance too; the model also computes it in float64 and reports the rays whose
two decisions differ (`cut_disagree`): they lie within rounding of max_range and are ambiguous.

Cells.  Cell k of an axis is [k vs, (k + 1) vs) relative to the origin, grid index k + res / 2 (the floor rule of
GetVoxel, the hit voxel, collision, the EDT and CreateFromOccupancyGrid).

Per ray, the segment s -> e is classified in float64.  The crossing parameters t = (k vs - s_a) / (e_a - s_a) of every
axis are merged; each piece between two crossings names a crossed cell.  For a cell c the model computes its depth: the
largest x such that the segment meets c shrunk by x on every side over an interval of positive length (x < 0: c grown by
|x|), in closed form from the slab bounds (`depth`).  With the tolerance delta of the ray, a cell is
  - required when depth > delta (the segment passes through the cell shrunk by delta);
  - allowed when depth >= -delta (the segment comes within delta of the closed cell);
  - forbidden otherwise.
A cell touched only along a face, an edge or a corner has depth 0: allowed, not required.  Two rules of the walk on top:
  - the start cell floor(s / vs) is always on the ray's list (the walk lists it before its first step): required when s
    lies more than delta inside it, even if the ray is short or ends in it;
  - the end cell is never on the list otherwise (:119-121): a cell within delta of e is never required by this ray, and
    the cell of e is forbidden for it when e lies more than delta inside it and s more than delta outside it.
A ray of length 0 lists nothing.

The tolerance.  delta = C delta1 with
    delta1 = 2^-24 (|s|_inf + |e|_inf + vs + 2 L + sum_a (k_a + 1) (E_a + 4 vs)),
L the segment's length, E_a = |e_a - s_a| its extent and k_a = |floor(e_a / vs) - floor(s_a / vs)| the planes it steps
over on axis a.  The first three terms cover the float32 division and floor of the start and end cells and the rounding
of the first boundary and of ray = e - s; 2 L covers the direction's rounding (a relative 2^-23 of the position after
length L).  The sum is the drift of the walk's tmax_a += tdelta_a, measured as a position along axis a (times |ray_a|):
each of its k_a + 1 steps rounds tmax_a <= L + tdelta_a to half an ulp, at most 2^-24 (E_a + vs) along the axis, and
carries tdelta_a's own error, a relative 2^-22 (the divisions by length and by |ray_a|), at most 2^-22 vs.  That is a
worst case: it grows as the square of the cells per axis, so on a ray of 645 cells per axis at vs 1 delta is 0.3 vs.
C = DELTA_C (see its comment).  Each candidate cell's
depth / delta1 is its ratio: a listed cell with a negative ratio, or an unlisted one with a positive ratio, shows how far
off the walk was, in units of delta1 (`max_ratio`).

Per Insert (`check_insert`), with Occ the occupied cells (in the grid, of the hit rays' end points):
  - the free set F satisfies  U required_i \\ Occ  <=  F  <=  U allowed_i \\ Occ  over the cells inside the grid;
  - each cell changes once: Occ cells by prob_hit_log, F cells by prob_miss_log, both in float32 then clamped to
    [clamping_thres_min, clamping_thres_max]; a NaN (unknown) cell counts as 0; every other cell keeps its bits;
  - the bounds become the u16 min / max of the previous bounds and F U Occ.
F and Occ are read back from the grid before and after the call: a changed cell is occupied or free by its new value.
A cell whose update the clamp hides (free at clamping_thres_min, occupied at clamping_thres_max) cannot be observed and
is not held to either direction.  An end point within delta of a face may land in either cell: its neighbours across
that face (and, near an edge or a corner, across both or all three) are accepted for Occ too.  With `full=False` only the
rays given are modelled (a subset of the call): then only the lower bound  U required_i \\ Occ <= F  is checked.
"""
import numpy as np

U = 2.0 ** -24
# delta1 is a sum of worst-case terms, each taken at one unit; C = 4 covers the constants the analysis above rounds
# away (a few roundings per term) with a margin, and is not a fit.  The largest measured ratio of a listed cell's
# distance outside, or an unlisted cell's depth inside, to delta1 (printed as max_ratio) is 0.018 on the inputs
# of tests/test_oracle_occgrid64.py and 0.046 on those of tests/test_gpu_occgrid64.py.
DELTA_C = 4.0
RAY_CHUNK = 2048       # rays per vectorised pass of the classification
EXTRA_CAP = 4096       # listed cells outside every candidate checked by brute force over all rays (the rest: reported)


# known answers (name, start, end, free cells, occupied cell; unshifted cell coordinates, origin 0) with vs = 0.25: every
# coordinate, crossing and tie below is exact in float32
KNOWN_ANSWERS = [
    # a ray in the grid plane z = 0.5 takes the floor cell z = 2
    ("plane z", (0.125, 0.125, 0.5), (1.125, 0.375, 0.5), [(0, 0, 2), (1, 0, 2), (2, 0, 2), (2, 1, 2), (3, 1, 2)], (4, 1, 2)),
    # along x in the planes y = 0.5 and z = 0.5
    ("line yz", (0.125, 0.5, 0.5), (1.125, 0.5, 0.5), [(0, 2, 2), (1, 2, 2), (2, 2, 2), (3, 2, 2)], (4, 2, 2)),
    # through grid edges: tmax_x == tmax_y at every crossing, the walk steps y first
    ("edges", (0.125, 0.125, 0.375), (0.875, 0.875, 0.375),
     [(0, 0, 1), (0, 1, 1), (1, 1, 1), (1, 2, 1), (2, 2, 1), (2, 3, 1)], (3, 3, 1)),
    # through grid corners: a three-way tie steps z, then y, then x
    ("corners", (0.125, 0.125, 0.125), (0.625, 0.625, 0.625),
     [(0, 0, 0), (0, 0, 1), (0, 1, 1), (1, 1, 1), (1, 1, 2), (1, 2, 2)], (2, 2, 2)),
    # a start on the face x = 0.5 going down leaves cell 2 at t = 0
    ("start on face", (0.5, 0.125, 0.125), (0.125, 0.875, 0.125), [(2, 0, 0), (1, 0, 0), (1, 1, 0), (1, 2, 0), (0, 2, 0)],
     (0, 3, 0)),
    # an end on a face: going up it is the upper cell's, going down the walk stops on entering it
    ("end on face up", (0.125, 0.125, 0.125), (1.0, 0.125, 0.125), [(0, 0, 0), (1, 0, 0), (2, 0, 0), (3, 0, 0)], (4, 0, 0)),
    ("end on face down", (1.125, 0.125, 0.125), (0.5, 0.125, 0.125), [(4, 0, 0), (3, 0, 0)], (2, 0, 0)),
    # a ray inside one cell lists its start cell, which is occupied
    ("one cell", (0.3, 0.3, 0.3), (0.4, 0.45, 0.35), [], (1, 1, 1)),
]


def form_rays(points, viewpoint, origin, max_range=-1.0):
    """the Insert's inputs as the library forms them (occgrid.cu::occ_range_kernel, float32) -> dict: s[3], e[n, 3]
    (float64 copies of float32 values, relative to the origin), hit[n], cut_disagree (count of rays whose float64 and
    float32 max_range decisions differ)"""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    v = np.asarray(viewpoint, np.float32).reshape(3)
    o = np.asarray(origin, np.float32).reshape(3)
    mr = np.float32(max_range)
    d = p - v
    dist = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    hit = np.full(len(p), True) if mr < 0 else dist <= mr
    with np.errstate(divide="ignore", invalid="ignore"):
        cut = v + (d / dist[:, None]) * mr
    r = np.where(hit[:, None], p, np.where((dist == 0)[:, None], v, cut)).astype(np.float32)
    dist64 = np.linalg.norm(p.astype(np.float64) - v.astype(np.float64), axis=1)
    hit64 = np.full(len(p), True) if mr < 0 else dist64 <= float(mr)
    return dict(s=(v - o).astype(np.float64), e=(r - o).astype(np.float64), hit=hit,
                cut_disagree=int((hit != hit64).sum()))


def depth(s, D, c, vs):
    """largest x such that s + t D, t in [0, 1], meets cell c (int [m, 3]) shrunk by x on every side over a t interval of
    positive length (negative: grown).  s, D [m, 3] float64 -> [m]"""
    lo = c * vs - s                          # the cell's faces relative to s
    hi = (c + 1) * vs - s
    moving = D != 0
    with np.errstate(divide="ignore", invalid="ignore"):
        a0 = np.where(moving, np.minimum(lo / D, hi / D), 0.0)   # t interval of the slab
        a1 = np.where(moving, np.maximum(lo / D, hi / D), 0.0)
        q = np.where(moving, 1.0 / np.abs(D), 0.0)              # d t / d x of each slab bound
        x = np.where(moving, np.inf, np.minimum(-lo, hi)).min(1)   # a still axis: s's distance inside the slab
        for j in range(3):
            for k in range(3):                                   # lower bound of slab j <= upper bound of slab k
                x = np.minimum(x, np.where(moving[:, j] & moving[:, k], (a1[:, k] - a0[:, j]) / (q[:, j] + q[:, k]), np.inf))
            x = np.minimum(x, np.where(moving[:, j], (1.0 - a0[:, j]) * np.abs(D[:, j]), np.inf))   # ... <= t = 1
            x = np.minimum(x, np.where(moving[:, j], a1[:, j] * np.abs(D[:, j]), np.inf))           # t = 0 <= ...
    return x


def _inside(p, c, vs):
    """how far p [m, 3] lies inside cell c [m, 3] (L_inf; negative: outside) -> [m]"""
    return np.minimum(p - c * vs, (c + 1) * vs - p).min(1)


def crossed_cells(s, e, vs):
    """-> (ray [m] int64, cell [m, 3] int64, k [n] cells crossed per ray): the cells of the float64 walk of every
    segment s -> e[i] (e [n, 3]); a tie between axes gives a piece of zero length, which is dropped, or of a few ulps"""
    e = np.asarray(e, np.float64).reshape(-1, 3)
    n = len(e)
    D = e - s
    out_r, out_c = [], []
    k = np.zeros(n, np.int64)
    for b in range(0, n, RAY_CHUNK):
        E, Dc = e[b:b + RAY_CHUNK], D[b:b + RAY_CHUNK]
        m = len(E)
        S = np.broadcast_to(s, E.shape)
        lo, hi = np.minimum(S, E) / vs, np.maximum(S, E) / vs
        k0 = np.floor(lo) + 1
        cnt = np.maximum(np.ceil(hi) - 1 - k0 + 1, 0).astype(np.int64)      # planes strictly between the end points
        ts = [np.zeros((m, 1)), np.ones((m, 1))]
        with np.errstate(divide="ignore", invalid="ignore"):
            for a in range(3):
                w = int(cnt[:, a].max(initial=0))
                if w == 0:
                    continue
                j = np.arange(w)[None, :]
                t = ((k0[:, a:a + 1] + j) * vs - S[:, a:a + 1]) / Dc[:, a:a + 1]
                ts.append(np.where(j < cnt[:, a:a + 1], t, 1.0))
        T = np.sort(np.concatenate(ts, 1), 1)
        t0, t1 = T[:, :-1], T[:, 1:]
        keep = (t1 > t0) & (np.linalg.norm(Dc, axis=1) > 0)[:, None]
        ri, pi = np.nonzero(keep)
        mid = 0.5 * (t0[ri, pi] + t1[ri, pi])
        cell = np.floor((S[ri] + mid[:, None] * Dc[ri]) / vs).astype(np.int64)
        # neighbouring pieces of one cell (a crossing of a few ulps back and forth): keep one
        first = np.ones(len(ri), bool)
        first[1:] = (ri[1:] != ri[:-1]) | (cell[1:] != cell[:-1]).any(1)
        ri, cell = ri[first], cell[first]
        k[b:b + m] = np.bincount(ri, minlength=m)
        out_r.append(ri + b)
        out_c.append(cell)
    return np.concatenate(out_r) if out_r else np.zeros(0, np.int64), \
        np.concatenate(out_c) if out_c else np.zeros((0, 3), np.int64), k


def delta1(s, e, vs, k=None):
    """the module's delta1 of every segment s -> e[i] -> [n] (k, the cells crossed, is not needed: the per-axis plane
    counts are)"""
    e = np.asarray(e, np.float64).reshape(-1, 3)
    E = np.abs(e - s)
    L = np.linalg.norm(e - s, axis=1)
    ka = np.abs(np.floor(e / vs) - np.floor(s / vs))             # planes the walk steps over, per axis
    return U * (np.abs(s).max() + np.abs(e).max(1) + vs + 2 * L + ((ka + 1) * (E + 4 * vs)).sum(1))


def classify(s, e, vs, C=DELTA_C, ray=None, cell=None):
    """every candidate (ray, cell) pair of the segments s -> e[i] -> dict of arrays over the pairs: ray, cell [m, 3]
    (unshifted cell coordinates), req, alw, ratio (depth / delta1; NaN where a start or end rule decides), and per ray
    d1 and k.  By default the candidates are the crossed cells; (ray, cell) may name others (the brute-force check)."""
    e = np.asarray(e, np.float64).reshape(-1, 3)
    r0, c0, k = crossed_cells(s, e, vs)
    if ray is None:
        ray, cell = r0, c0
    d1 = delta1(s, e, vs, k)
    D = e - s
    L = np.linalg.norm(D, axis=1)
    S = np.broadcast_to(s, (len(ray), 3))
    dep = depth(S, D[ray], cell, vs)
    dl = C * d1[ray]
    req = dep > dl
    alw = dep >= -dl
    special = np.zeros(len(ray), bool)
    # the start cell is always listed
    scell = np.floor(s / vs).astype(np.int64)
    is_start = (cell == scell).all(1)
    s_in = _inside(S, cell, vs)                      # s's depth in the candidate cell
    st = is_start & (s_in > dl) & (L[ray] > 0)
    req |= st
    special |= st
    # the end cell is not listed
    e_in = _inside(e[ray], cell, vs)
    near_end = e_in >= -dl
    req &= ~near_end | st
    special |= near_end & ~st
    ecell = np.floor(e[ray] / vs).astype(np.int64)
    forb = (cell == ecell).all(1) & (e_in > dl) & (s_in < -dl)
    alw &= ~forb
    alw &= L[ray] > 0
    req &= L[ray] > 0
    ratio = np.where(special, np.nan, dep / d1[ray])
    return dict(ray=ray, cell=cell, req=req, alw=alw, ratio=ratio, d1=d1, k=k)


def _lin(g, res):
    return (g[:, 0] * res + g[:, 1]) * res + g[:, 2]


def _in_grid(g, res):
    return ((g >= 0) & (g < res)).all(1)


def _group(lin, *vals):
    """per distinct lin: (ulin, max of each val)"""
    if len(lin) == 0:
        return (np.zeros(0, np.int64),) + tuple(np.zeros(0, v.dtype) for v in vals)
    o = np.argsort(lin, kind="stable")
    ls = lin[o]
    head = np.ones(len(ls), bool)
    head[1:] = ls[1:] != ls[:-1]
    st = np.flatnonzero(head)
    out = [ls[st]]
    for v in vals:
        vv = v[o]
        if vv.dtype == bool:
            out.append(np.maximum.reduceat(vv.astype(np.int8), st).astype(bool))
        else:
            out.append(np.fmax.reduceat(vv, st))
    return tuple(out)


def ray_sets(s, e, vs, C=DELTA_C):
    """one ray's (required, allowed) cell sets (unshifted cell coordinates, sets of tuples)"""
    r = classify(np.asarray(s, np.float64), np.asarray(e, np.float64).reshape(1, 3), vs, C)
    req = {tuple(c) for c in r["cell"][r["req"]].tolist()}
    alw = set()
    c = r["cell"]
    # the allowed cells that the walk does not cross: the 26 neighbours of the crossed ones
    nb = np.array([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)], np.int64)
    cand = np.unique((c[:, None, :] + nb[None]).reshape(-1, 3), axis=0)
    if len(cand):
        q = classify(np.asarray(s, np.float64), np.asarray(e, np.float64).reshape(1, 3), vs, C,
                     ray=np.zeros(len(cand), np.int64), cell=cand)
        alw = {tuple(x) for x in cand[q["alw"]].tolist()}
    return req, alw


def _f32_update(before, inc, cmin, cmax):
    b = np.where(np.isnan(before), np.float32(0), before).astype(np.float32)
    return np.minimum(np.maximum((b + np.float32(inc)).astype(np.float32), np.float32(cmin)), np.float32(cmax))


def check_insert(before, after, bounds_before, bounds_after, points, viewpoint, origin, vs, res, max_range=-1.0,
                 params=(-2.0, 3.5, 0.85, -0.4), full=True, C=DELTA_C, label=""):
    """assert the module's Insert rules for one call that took the dense grid `before` to `after` (float32 [res^3], NaN
    unknown) and the bounds (u16[6] min xyz, max xyz) from bounds_before to bounds_after.  params = (clamping_thres_min,
    clamping_thres_max, prob_hit_log, prob_miss_log).  -> dict of counts and the largest measured ratio (printed)"""
    vs = float(np.float32(vs))
    cmin, cmax, hit_log, miss_log = params
    half = res // 2
    before = np.asarray(before, np.float32).reshape(-1)
    after = np.asarray(after, np.float32).reshape(-1)
    R = form_rays(points, viewpoint, origin, max_range)
    s, e, hit = R["s"], R["e"], R["hit"]
    up_hit = _f32_update(before, hit_log, cmin, cmax)
    up_miss = _f32_update(before, miss_log, cmin, cmax)
    changed = np.flatnonzero(after.view(np.uint32) != before.view(np.uint32))
    ch_occ = after[changed].view(np.uint32) == up_hit[changed].view(np.uint32)
    ch_free = after[changed].view(np.uint32) == up_miss[changed].view(np.uint32)
    bad = ~(ch_occ | ch_free)
    assert not bad.any(), "%s: %d cells changed by neither increment; first %d: %r -> %r" % (
        label, int(bad.sum()), int(changed[bad][0]), before[changed[bad][0]], after[changed[bad][0]])
    occ_obs, free_obs = changed[ch_occ], changed[ch_free & ~ch_occ]
    hide_occ = up_hit.view(np.uint32) == before.view(np.uint32)       # an occupied update the clamp hides
    hide_free = up_miss.view(np.uint32) == before.view(np.uint32)

    # the candidate cells of every ray, in chunks: grid lin index (in the grid only), req, alw, ratio
    parts, d1 = [], np.zeros(len(e))
    for b in range(0, len(e), 8 * RAY_CHUNK):
        r = classify(s, e[b:b + 8 * RAY_CHUNK], vs, C)
        d1[b:b + 8 * RAY_CHUNK] = r["d1"]
        gi = r["cell"] + half
        ing = _in_grid(gi, res)
        parts.append((_lin(gi[ing], res), r["req"][ing], r["alw"][ing], r["ratio"][ing], len(r["ray"])))
    n_cand = sum(x[4] for x in parts)
    lin, req_c, alw_c, rat_c = (np.concatenate([x[i] for x in parts]) for i in range(4))
    del parts

    # Occ: the floor cells of the hit end points, either side of a face within delta of it
    eh = e[hit]
    cell = np.floor(eh / vs).astype(np.int64)
    dl_hit = C * d1[hit]
    frac = eh / vs - cell
    lo_amb = frac * vs <= dl_hit[:, None]
    hi_amb = (1 - frac) * vs <= dl_hit[:, None]
    amb = (lo_amb | hi_amb).any(1)
    g = cell + half
    sure = g[~amb & _in_grid(g, res)]
    occ_sure = np.unique(_lin(sure, res))
    alts = []
    for off in np.array([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)]):
        m = ((off == 0) | ((off < 0) & lo_amb) | ((off > 0) & hi_amb)).all(1)
        alts.append(g[m] + off)
    alts = np.concatenate(alts)
    occ_alw = np.unique(_lin(alts[_in_grid(alts, res)], res))
    miss_occ = np.setdiff1d(occ_sure[~hide_occ[occ_sure]], occ_obs)
    assert len(miss_occ) == 0, "%s: %d occupied cells not updated; first grid index %r" % (
        label, len(miss_occ), np.unravel_index(miss_occ[0], (res,) * 3))
    extra_occ = np.setdiff1d(occ_obs, occ_alw) if full else np.zeros(0, np.int64)
    assert len(extra_occ) == 0, "%s: %d cells updated as occupied that hold no hit end point; first %r" % (
        label, len(extra_occ), np.unravel_index(extra_occ[0], (res,) * 3))
    occ_set = np.union1d(occ_obs, occ_sure)

    # F
    ulin, req_u, alw_u, rat_u = _group(lin, req_c, alw_c, rat_c)
    del lin, req_c, alw_c, rat_c
    notocc = ~np.isin(ulin, occ_set)
    need = ulin[req_u & notocc]
    missing = np.setdiff1d(need, free_obs)
    missing = missing[~hide_free[missing]]
    in_free = np.isin(ulin, free_obs)
    max_ratio = 0.0
    unlisted = notocc & ~in_free & ~hide_free[ulin] & ~np.isnan(rat_u)
    if unlisted.any():
        max_ratio = max(max_ratio, float(rat_u[unlisted].max(initial=0.0)))
    listed = in_free & ~np.isnan(rat_u)
    if listed.any():
        max_ratio = max(max_ratio, float((-rat_u[listed]).max(initial=0.0)))
    extra_n = 0
    extra_ok = np.zeros(0, np.int64)
    if full:
        extra = np.setdiff1d(free_obs, ulin[alw_u])
        extra_n = len(extra)
        chk = extra[:EXTRA_CAP]
        if len(chk):
            ok = np.zeros(len(chk), bool)
            best = np.full(len(chk), -np.inf)
            cc = np.stack(np.unravel_index(chk, (res,) * 3), 1).astype(np.int64) - half
            n = len(e)
            for b in range(0, n, max(1, (1 << 20) // len(chk))):
                rr = np.arange(b, min(n, b + max(1, (1 << 20) // len(chk))))
                ray = np.repeat(rr, len(chk))
                cl = np.tile(cc, (len(rr), 1))
                q = classify(s, e, vs, C, ray=ray, cell=cl)
                ok |= q["alw"].reshape(len(rr), len(chk)).any(0)
                best = np.fmax(best, q["ratio"].reshape(len(rr), len(chk)).max(0))
            listed_out, extra_ok = chk[~ok], chk[ok]
            if len(best):
                max_ratio = max(max_ratio, float(np.nan_to_num(-best, nan=0.0, posinf=np.inf).max(initial=0.0)))
            extra = np.concatenate([listed_out, extra[EXTRA_CAP:]])
        extra_n = len(extra)
        info_extra = extra
    else:
        info_extra = np.zeros(0, np.int64)
    info = dict(rays=len(e), hits=int(hit.sum()), crossed=n_cand, required=len(need), free=len(free_obs),
                occupied=len(occ_obs), missing=len(missing), outside=extra_n, cut_disagree=R["cut_disagree"],
                ambiguous_ends=int(amb.sum()), max_ratio=max_ratio)
    print("%s occgrid64: %s" % (label, info))
    assert len(missing) == 0, "%s: %d required cells not freed; first grid index %r" % (
        label, len(missing), np.unravel_index(missing[0], (res,) * 3))
    assert extra_n == 0, "%s: %d freed cells farther than delta from every ray; first grid index %r" % (
        label, extra_n, np.unravel_index(info_extra[0], (res,) * 3))

    # each cell changed once, by its own rule (checked above), and the bounds
    bb = np.asarray(bounds_before, np.int64).reshape(6)
    ba = np.asarray(bounds_after, np.int64).reshape(6)
    touched_min = np.union1d(occ_obs, np.union1d(free_obs, need))          # surely in F U Occ (or hidden)
    touched_max = np.union1d(np.union1d(occ_alw, ulin[alw_u & notocc]), extra_ok) if full else touched_min
    def _mm(lins):
        if len(lins) == 0:
            return np.full(3, 1 << 30), np.full(3, -1)
        x = np.stack(np.unravel_index(lins, (res,) * 3), 1)
        return x.min(0), x.max(0)
    lo_in, hi_in = _mm(touched_min)
    lo_out, hi_out = _mm(touched_max)
    if full:
        assert (ba[:3] >= np.minimum(bb[:3], lo_out)).all() and (ba[3:] <= np.maximum(bb[3:], hi_out)).all(), \
            "%s: bounds %r outside the allowed cells' box %r %r (before %r)" % (label, ba, lo_out, hi_out, bb)
    assert (ba[:3] <= np.minimum(bb[:3], lo_in)).all() and (ba[3:] >= np.maximum(bb[3:], hi_in)).all(), \
        "%s: bounds %r do not cover the updated cells' box %r %r (before %r)" % (label, ba, lo_in, hi_in, bb)
    return info


def cell_of(point, origin, vs, res):
    """the grid index of a point by the floor rule, in float64 -> (int64[3], distance to the nearest face in voxels)"""
    x = (np.asarray(point, np.float32).astype(np.float64) - np.asarray(origin, np.float32).astype(np.float64)) / \
        float(np.float32(vs))
    f = np.floor(x)
    return f.astype(np.int64) + res // 2, float(np.minimum(x - f, f + 1 - x).min())


def voxel_index(point, origin, vs, res):
    """GetVoxel's linear index (densegrid.inl:137-146): only the linear index is range-checked -> int or -1"""
    g, _ = cell_of(point, origin, vs, res)
    i = int((g[0] * res + g[1]) * res + g[2])
    return i if 0 <= i < res ** 3 else -1


def free_area_box(min_bound, max_bound, origin, vs, res):
    """SetFreeArea's box of grid indices (occupancygrid.cu:415-460), clipped to the grid -> (lo[3], hi[3])"""
    lo, _ = cell_of(min_bound, origin, vs, res)
    hi, _ = cell_of(max_bound, origin, vs, res)
    return np.maximum(lo, 0), np.minimum(hi, res - 1)
