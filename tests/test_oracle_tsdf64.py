"""CPU: ExtractPointCloud and Raycast of the UniformTSDFVolume restatement (oracle/tsdf.c) against the float64
restatement cupoch_b200/testing/tsdf64.py and against analytic fields.

Restatement parity.  Rows whose decision margin exceeds the row's slack must agree: the same hit flags and crossings,
the colour of the same voxel (the written fields' RGB8 planes hold each voxel's indices, so a colour names its voxel),
and points and normals within these bounds, derived from float32 rounding (u = 2^-24):
  - ExtractPointCloud point: each coordinate is formed by at most four roundings of quantities below 2 L + |o|
    (L the length): 4 u (2 L + |o|).  Normal: a GetTSDFAt sample position is off by at most 3 u res voxels (p -+ half_gap
    rounded, p / vl, - 0.5), which moves a value by 2 per voxel at most, and the 8-term sum adds 10 u; the difference of
    two samples is then off by 2 (6 u res + 10 u) per axis, and a unit vector by sqrt(3) times that over |n|:
    u (16 res + 64) / |n| bounds it.  Colour: 4 u of the largest colour.
  - Raycast: the float32 march length is off by at most `drift` (tsdf64's bound) and a sample position by
    e = drift + 8 u (|t| + ts + |o|) (t the camera relative to the origin, ts the hit length).  That is the point bound;
    in voxel units plus the 4 u res of loc = vertex / vl + res / 2 it is the slack s the decision margins are compared
    with.  Normal: the six InterpolateTrilinearly samples move by s voxels together, so each difference is off by
    at most 2 * 2 s (a gradient of at most 2 per voxel on either side) plus 20 u: 2 sqrt(3) (4 s + 20 u) / |n|.
Rows at or under their slack are listed with their margins.  Every differing row must be one of them, and they stay
under 1 % of an image's rows (observed: at most 0.35 % of an image, 0.12 % over all the images here).
Observed worst error over bound: ExtractPointCloud points 0.31, normals 0.10; Raycast points 0.21, normals 0.009.

Analytic fields.  Planar f = clamp((n.x - c) / trunc, -1, 1) at the voxel centres, weight 1, trunc = 5 vl, so every
normal stencil reads unclamped values: ExtractPointCloud points lie on the plane to rounding (linear interpolation of a
linear field is exact), normals equal n, the crossing count equals the straddling centre pairs counted in integers, and a
centre exactly on the plane (f == 0) emits nothing on either side.  Raycast hits lie within (|n|_1 / 2) vl of the plane
(the march reads voxel-centre values at the samples' cells, up to half a voxel per axis away), normals equal n, and a
camera on the negative side never hits: a - to + crossing ends the march.  A written sphere of radius R: hits and
points within (sqrt(3) / 2) vl + vl^2 / R of it, normals within 2 vl / R radians of radial.

Geometry edges: odd resolutions (3, 5, 63, 129), origins off the voxel lattice, cameras outside each face, inside the
grid, inside the sphere and on a face of the entry box, axis-parallel rays along cell faces with a dyadic voxel length
(float32 and float64 are both exact and agree with no slack), grazing rays through an edge and a corner of the box,
steps shorter than a voxel and a thin shell stepped over, and a camera so far that len + step == len at entry: the
project's no-advance rule makes that a miss where float64 hits."""
import numpy as np
import pytest

from cupoch_b200.testing import tsdf64 as X
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import tsdf_py as T

U = X.EPS32
SLACK_FRACTION = 0.01


# ------------------------------------------------------------------------------------------------ fields and cameras
def centres(res, length, origin):
    """float64 voxel centres [res, res, res, 3]: origin + vl (k - res / 2) + vl / 2"""
    vl = float(np.float32(length) / np.float32(res))
    k = (np.arange(res) - res // 2 + 0.5) * vl
    o = np.asarray(origin, np.float32).astype(np.float64)
    X_, Y_, Z_ = np.meshgrid(k + o[0], k + o[1], k + o[2], indexing="ij")
    return np.stack([X_, Y_, Z_], -1)


def written(res, length, trunc, sdf, origin=(0.0, 0.0, 0.0), ct=T.RGB8):
    """a volume whose tsdf is clamp(sdf(centre) / trunc, -1, 1), weight 1; the RGB8 planes hold the voxel's (x, y, z)"""
    vol = T.Volume(length, res, trunc, ct, origin)
    vol.tw[:, 0] = np.clip(sdf(centres(res, length, origin)) / np.float64(np.float32(trunc)), -1, 1).reshape(-1)
    vol.tw[:, 1] = 1.0
    if ct == T.RGB8:
        vol.col[:] = np.stack(np.meshgrid(*[np.arange(res)] * 3, indexing="ij"), 0).reshape(3, -1)
        vol.names_voxels = True
    return vol


def sphere_sdf(R, c=(0.0, 0.0, 0.0)):
    return lambda x: np.linalg.norm(x - np.asarray(c), axis=-1) - R


def plane_sdf(n, c):
    return lambda x: x @ np.asarray(n, np.float64) - c


def look_at(eye, target, w, h, f, up=(0.0, 0.0, 1.0)):
    """(K, world-to-camera E) of a pinhole camera at eye looking at target"""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    zc = (target - eye) / np.linalg.norm(target - eye)
    up = np.asarray(up, np.float64)
    if abs(zc @ up) > 0.99:
        up = np.array([0.0, 1.0, 0.0])
    xc = np.cross(zc, up)
    xc /= np.linalg.norm(xc)
    R = np.stack([xc, np.cross(zc, xc), zc])
    E = np.eye(4)
    E[:3, :3], E[:3, 3] = R, -R @ eye
    K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]])
    return K.astype(np.float32), E.astype(np.float32)


def axis_camera(eye, axis, sign):
    """a 1 x 1 camera at eye whose one pixel looks exactly along sign * e_axis (a permutation extrinsic)"""
    E = np.zeros((4, 4), np.float32)
    others = [a for a in range(3) if a != axis]
    E[0, others[0]] = E[1, others[1]] = 1.0
    E[2, axis] = sign
    E[3, 3] = 1.0
    E[:3, 3] = -E[:3, :3] @ np.asarray(eye, np.float32)
    return np.float32([[1, 0, 0], [0, 1, 0], [0, 0, 1]]), E


# ------------------------------------------------------------------------------------------------ comparisons
def vl_of(vol):
    return float(vol.voxel_length)


def check_points(vol, p=None, n=None, c=None):
    """(vol: an oracle Volume, or anything with its attributes and `block` as tsdf64 takes it)
    the extraction (the oracle's unless given) against extract_point_cloud64 -> (restatement, worst error / bound)"""
    if p is None:
        p, n, c = vol.extract_point_cloud()
    r = X.extract_point_cloud64(vol.tw, vol.col, vol.length, vol.res, vol.origin, vol.ct, getattr(vol, "block", None))
    assert not (r.margin <= 0).any()  # no underflowing product or normal in these fields: the crossings are decided exactly
    assert len(p) == len(r.rows)
    worst = {"points": 0.0, "normals": 0.0}
    if not len(p):
        return r, worst
    o = np.abs(vol.origin.astype(np.float64)).max()
    tol_p = 4 * U * (2 * vol.length + o)
    tol_n = U * (16 * vol.res + 64) / r.nscale
    ep = np.abs(p - r.points).max(1)
    en = np.abs(n - r.normals).max(1)
    assert np.all(ep <= tol_p), ep.max()
    assert np.all(en <= tol_n), (en / tol_n).max()
    if vol.ct != T.NO_COLOR:
        assert np.all(np.abs(c - r.colors) <= 4 * U * max(1.0, np.abs(r.colors).max()))
    worst["points"], worst["normals"] = float(ep.max() / tol_p), float((en / tol_n).max())
    return r, worst


def camera_t(E, origin):
    E = np.asarray(E, np.float32).astype(np.float64).reshape(4, 4)
    return -E[:3, :3].T @ E[:3, 3] - np.asarray(origin, np.float32).astype(np.float64)


def check_rays(vol, K, E, w, h, trunc, rows=None, max_listed=None):
    """the raycast (the oracle's unless rows = (points, normals, colours) with NaN misses) against raycast64.
    max_listed: the most under-slack rows allowed (default 1 % of the pixels)
    -> (restatement, the under-slack rows as [(pixel, margin)], worst error / bound)"""
    if rows is None:
        rows = vol.raycast(K, E, w, h, trunc, False)
    pp, nn, cc = (np.asarray(a, np.float32) for a in rows)
    hit = np.isfinite(pp[:, 0])
    r = X.raycast64(vol.tw, vol.col, vol.length, vol.res, vol.origin, vol.ct, K, E, trunc, w, h, getattr(vol, "block", None))
    vl = vl_of(vol)
    tn = np.linalg.norm(camera_t(E, vol.origin))
    o = np.abs(vol.origin.astype(np.float64)).max()
    ts = np.where(r.hit, r.ts, 0.0)
    e = r.drift + 8 * U * (tn + ts + o)
    s = e / vl + 4 * U * vol.res
    low = r.margin <= s
    both = hit & r.hit
    bad = hit != r.hit
    ep = np.where(both, np.abs(pp - r.points).max(1), 0.0)
    tol_n = 2 * np.sqrt(3) * (4 * s + 20 * U) / np.where(both, r.nscale, 1.0)
    en = np.where(both, np.abs(nn - r.normals).max(1), 0.0)
    bad |= both & ((ep > e) | (en > tol_n))
    if getattr(vol, "names_voxels", False):  # the colour names the voxel it was read from
        bad |= both & np.any(np.round(np.where(both[:, None], cc, 0) * 255).astype(np.int64) != r.voxel, axis=1)
    elif vol.ct != T.NO_COLOR:  # the same voxel's colour, divided by 255 in float32 or float64
        bad |= both & np.any(np.abs(np.where(both[:, None], cc - r.colors, 0)) > 2 * U * np.abs(np.nan_to_num(r.colors)), axis=1)
    listed = [(int(i), float(r.margin[i])) for i in np.nonzero(low)[0]]
    assert not (bad & ~low).any(), [(int(i), float(r.margin[i]), float(s[i])) for i in np.nonzero(bad & ~low)[0]][:10]
    assert len(listed) <= (SLACK_FRACTION * w * h + 1 if max_listed is None else max_listed), listed[:20]
    ok = both & ~low
    worst = {"points": float((ep[ok] / e[ok]).max()) if ok.any() else 0.0,
             "normals": float((en[ok] / tol_n[ok]).max()) if ok.any() else 0.0}
    return r, listed, worst


def within(hit_points, dist, bound):
    return np.all(np.abs(dist(hit_points.astype(np.float64))) <= bound)


# ------------------------------------------------------------------------------------------------ restatement parity
@pytest.mark.parametrize("res", [63, 64])
def test_sphere_views_match_the_float64_restatement(res):
    trunc, w, h = 0.08, 96, 72
    vol = T.Volume(2.0, res, trunc, T.RGB8, origin=(0.013, -0.021, 0.007))
    rng = np.random.default_rng(res)
    cams = ring_cameras(6, w, h)
    for K, E in cams:
        vol.integrate(sphere_depth(K, E, w, h, 0.6), rng.integers(0, 256, (h, w, 3), dtype=np.uint8), K, E)
    r, _ = check_points(vol)
    assert len(r.rows) > 3000
    for K, E in cams[:3] + ring_cameras(1, w, h, 0.9):
        ray, _, _ = check_rays(vol, K, E, w, h, trunc)
        assert ray.hit.sum() > 0.1 * w * h


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_smooth_fields_match_the_float64_restatement(seed):
    rng = np.random.default_rng(seed)
    res = (33, 40, 47)[seed]
    freq = rng.normal(0, 3.0, (3, 3))
    phase = rng.uniform(0, 2 * np.pi, 3)

    def sdf(x):
        return 0.25 * sum(np.sin(x @ freq[i] + phase[i]) for i in range(3)) + 0.05

    vol = written(res, 2.0, 0.12, sdf, origin=tuple(rng.uniform(-0.05, 0.05, 3)))
    r, _ = check_points(vol)
    assert len(r.rows) > 500
    hits = 0
    for k in range(4):
        eye = rng.normal(size=3)
        eye *= 2.5 / np.linalg.norm(eye)
        K, E = look_at(eye, rng.uniform(-0.3, 0.3, 3), 64, 48, 50.0)
        ray, _, _ = check_rays(vol, K, E, 64, 48, 0.12)
        hits += ray.hit.sum()
    assert hits > 1000


# ------------------------------------------------------------------------------------------------ planar fields
NORMALS = {"axis": (0.0, 0.0, 1.0), "diagonal": (1.0, 1.0, 0.0), "corner": (1.0, 1.0, 1.0), "random": (0.31, -0.72, 0.55)}


def plane_case(nkind, ckind, res=32, length=2.0):
    """(volume, unit normal, c): vl = 1 / 16 is dyadic, so the centres and c below are exact"""
    n = np.asarray(NORMALS[nkind], np.float64)
    n /= np.linalg.norm(n)
    vl = length / res
    ax = int(np.argmax(np.abs(n)))
    if ckind == "random":
        c = 0.1 * np.sqrt(2) - 0.037
    elif ckind == "centre":  # through the centre of voxel (h + 1, h + 1, h + 1)
        c = float(n @ np.full(3, 1.5 * vl))
    else:  # through a cell face: the one between centres h and h + 1 on the dominant axis
        p = np.full(3, 0.5 * vl)
        p[ax] = vl
        c = float(n @ p)
    vol = written(res, length, 5 * vl, plane_sdf(n, c))
    return vol, n, c


def straddling_pairs(vol):
    """ExtractPointCloud's crossing count from the field's signs: pairs (k, k + e_a) of band voxels with k interior,
    k_a + 1 < res - 1 and signs of opposite strict sign (a 0 straddles nothing)"""
    res = vol.res
    s = np.sign(vol.tw[:, 0].astype(np.float64)).astype(np.int64).reshape(res, res, res)
    band = (np.abs(vol.tw[:, 0]) < 0.98).reshape(res, res, res)
    total = 0
    inner = slice(1, res - 1)
    for a in range(3):
        lo = [inner] * 3
        hi = [inner] * 3
        lo[a], hi[a] = slice(1, res - 2), slice(2, res - 1)
        total += int(np.sum((s[tuple(lo)] * s[tuple(hi)] == -1) & band[tuple(lo)] & band[tuple(hi)]))
    return total


@pytest.mark.parametrize("ckind", ["random", "centre", "face"])
@pytest.mark.parametrize("nkind", list(NORMALS))
def test_planar_fields_extract_exactly(nkind, ckind):
    vol, n, c = plane_case(nkind, ckind)
    p, nrm, col = vol.extract_point_cloud()
    assert len(p) == straddling_pairs(vol)
    if nkind == "axis" and ckind == "centre":
        # the plane runs through a layer of centres: f == 0 there, and 0 straddles nothing on either side
        assert len(p) == 0 and (vol.tw[:, 0] == 0).sum() == 32 * 32
        return
    assert len(p) > 100
    assert within(p, plane_sdf(n, c), 4 * U * 2 * vol.length)
    assert np.all(np.abs(nrm - n) <= 64 * U * vol.res)
    check_points(vol, p, nrm, col)


@pytest.mark.parametrize("ckind", ["random", "face"])
@pytest.mark.parametrize("nkind", list(NORMALS))
def test_planar_fields_raycast_on_the_plane(nkind, ckind):
    vol, n, c = plane_case(nkind, ckind)
    vl, trunc, w, h = vl_of(vol), float(vol.trunc), 48, 36
    side = np.cross(n, [0.3, 0.5, 0.8])
    K, E = look_at(2.5 * n + 0.2 * side, -0.3 * side, w, h, 30.0)
    rows = vol.raycast(K, E, w, h, trunc, False)
    p, nrm = rows[0], rows[1]
    hit = np.isfinite(p[:, 0])
    assert hit.sum() > 0.25 * w * h
    bound = 0.5 * np.abs(n).sum() * vl + 8 * U * 4
    assert within(p[hit], plane_sdf(n, c), bound)
    assert np.all(np.abs(nrm[hit] - n) <= 64 * U * vol.res)
    check_rays(vol, K, E, w, h, trunc, rows)
    # from the negative side the march meets - to + first, which ends it
    K2, E2 = look_at(-2.5 * n + 0.2 * side, -0.3 * side, w, h, 30.0)
    rows2 = vol.raycast(K2, E2, w, h, trunc, False)
    assert not np.isfinite(rows2[0][:, 0]).any()
    ray, _, _ = check_rays(vol, K2, E2, w, h, trunc, rows2)
    assert not ray.hit.any()


# ------------------------------------------------------------------------------------------------ a written sphere
@pytest.mark.parametrize("res", [64, 65])
def test_written_sphere_is_found_within_a_voxel(res):
    R, length = 0.6, 2.0
    vol = written(res, length, 0.1, sphere_sdf(R), origin=(0.011, 0.0, -0.017))
    vl = vl_of(vol)
    bound = np.sqrt(3) / 2 * vl + vl * vl / R
    p, n, _ = vol.extract_point_cloud()
    assert len(p) > 5000
    radial = p.astype(np.float64) / np.linalg.norm(p.astype(np.float64), axis=1)[:, None]
    assert within(p, sphere_sdf(R), bound)
    assert np.all(np.arccos(np.clip((n * radial).sum(1), -1, 1)) <= 2 * vl / R)
    check_points(vol, p, n, _)
    for K, E in ring_cameras(3, 64, 48) + ring_cameras(1, 64, 48, 0.9):
        rows = vol.raycast(K, E, 64, 48, 0.1, False)
        hp, hn = rows[0], rows[1]
        hit = np.isfinite(hp[:, 0])
        assert hit.sum() > 300
        assert within(hp[hit], sphere_sdf(R), bound)
        rad = hp[hit].astype(np.float64) / np.linalg.norm(hp[hit].astype(np.float64), axis=1)[:, None]
        assert np.all(np.arccos(np.clip((hn[hit] * rad).sum(1), -1, 1)) <= 2 * vl / R)
        check_rays(vol, K, E, 64, 48, 0.1, rows)


# ------------------------------------------------------------------------------------------------ geometry edges
ODD = [3, 5, 63, 129]


def odd_volume(res):
    """a written sphere filling about 60 % of a 2 m grid at an origin off the voxel lattice"""
    return written(res, 2.0, max(0.1, 2.5 * 2.0 / res), sphere_sdf(0.6), origin=(0.0123, -0.0311, 0.0057))


@pytest.mark.parametrize("res", ODD)
def test_odd_resolutions_match_the_float64_restatement(res):
    vol = odd_volume(res)
    r, _ = check_points(vol)
    w, h = 40, 30
    hits = sum(check_rays(vol, K, E, w, h, float(vol.trunc))[0].hit.sum() for K, E in ring_cameras(3, w, h))
    if res == 3:
        # one interior voxel, whose +1 neighbour is never interior; and no loc -+ 1 fits [1, 2)
        assert len(r.rows) == 0 and hits == 0
    elif res >= 63:
        assert len(r.rows) > 1000 and hits > 600


def six_faces_inside_and_on_the_box(vol):
    """cameras outside each of the six faces, inside the grid, inside the sphere and exactly on the entry box's low-x
    face: (name, K, E)"""
    out = []
    for a in range(3):
        for sgn in (-1, 1):
            eye = np.zeros(3)
            eye[a] = 2.5 * sgn
            eye += [0.05, -0.07, 0.03]
            out.append(("face%d%+d" % (a, sgn),) + look_at(eye, np.zeros(3), 40, 30, 30.0))
    out.append(("inside grid",) + look_at([0.85, 0.1, -0.2], np.zeros(3), 40, 30, 30.0))
    out.append(("inside sphere",) + look_at([0.1, 0.05, 0.0], [1.0, 0.3, 0.2], 40, 30, 20.0))
    vl = vl_of(vol)
    lo = np.float32(vol.origin[0]) + np.float32(-(vol.res // 2)) * np.float32(vl)
    out.append(("on the box",) + look_at([float(lo), 0.1, 0.05], [0.0, 0.0, 0.0], 40, 30, 30.0))
    return out


def test_cameras_outside_every_face_inside_and_on_the_box():
    vol = odd_volume(63)
    for name, K, E in six_faces_inside_and_on_the_box(vol):
        ray, _, _ = check_rays(vol, K, E, 40, 30, float(vol.trunc))
        if name == "inside sphere":  # the march starts in negative tsdf: its first crossing is - to +, which ends it
            assert not ray.hit.any()
        else:
            assert ray.hit.sum() > 100, name


def axis_rays(res=32):
    """1 x 1 cameras looking exactly along -+x, -+y, -+z through lines on cell faces: (K, E) -- with vl = 1 / 16 and a
    zero origin every sample's grid coordinate on the other two axes is an exact integer"""
    vl = 2.0 / res
    out = []
    for axis in range(3):
        for sign in (-1, 1):
            for j in range(-6, 7, 3):
                for m in (-5, 0, 4):
                    eye = np.zeros(3)
                    eye[axis] = -2.5 * sign
                    others = [a for a in range(3) if a != axis]
                    eye[others[0]], eye[others[1]] = j * vl, m * vl
                    out.append(axis_camera(eye, axis, sign))
    return out


def test_axis_parallel_rays_along_cell_faces_agree_with_no_slack():
    vol = written(32, 2.0, 0.125, sphere_sdf(0.6))
    hits = 0
    for K, E in axis_rays():
        rows = vol.raycast(K, E, 1, 1, 0.125, False)
        r = X.raycast64(vol.tw, vol.col, vol.length, vol.res, vol.origin, vol.ct, K, E, 0.125, 1, 1)
        got = np.isfinite(rows[0][0, 0])
        assert got == r.hit[0]
        if got:
            hits += 1
            assert np.array_equal(np.round(rows[2][0] * 255).astype(np.int64), r.voxel[0])
            assert np.all(np.abs(rows[0][0] - r.points[0]) <= 16 * U)
            assert np.all(np.abs(rows[1][0] - r.normals[0]) <= 64 * U * 32 / r.nscale[0])
    assert hits >= 50


def test_grazing_rays_through_an_edge_and_a_corner_of_the_box():
    vol = odd_volume(63)
    vl = vl_of(vol)
    o = vol.origin.astype(np.float64)
    lo, hi = -(63 // 2) * vl, (63 - 1 - 63 // 2) * vl
    listed = 0
    for target in ([lo, lo, 0.0], [lo, hi, 0.2], [lo, lo, lo], [hi, hi, hi], [lo, hi, lo]):
        t = np.asarray(target) + o
        for eye in ([t[0] - 2.0, t[1] - 1.0, t[2] + 0.5], [t[0] + 0.3, t[1] - 2.0, t[2] - 0.7]):
            K, E = look_at(eye, t, 9, 9, 8.0)
            _, low, _ = check_rays(vol, K, E, 9, 9, float(vol.trunc), max_listed=9)
            listed += len(low)
    assert 0 < listed <= 0.05 * 10 * 81  # the central pixels graze the box


@pytest.mark.parametrize("field_trunc,ray_trunc", [(0.06, 0.04), (0.06, 0.5)])
def test_short_steps_and_a_thin_shell_stepped_over(field_trunc, ray_trunc):
    """ray_trunc 0.04: a step of 0.02, shorter than the 0.0317 voxel; 0.5: steps of 8 voxels over a shell 2 voxels
    thick, which most rays jump"""
    R = 0.6
    shell = lambda x: np.abs(np.linalg.norm(x, axis=-1) - R) - 0.0317  # noqa: E731
    vol = written(63, 2.0, field_trunc, shell if ray_trunc > 0.1 else sphere_sdf(R), origin=(0.0123, -0.0311, 0.0057))
    for K, E in ring_cameras(2, 48, 36):
        ray, _, _ = check_rays(vol, K, E, 48, 36, ray_trunc)
        if ray_trunc < 0.1:
            assert ray.hit.sum() > 300
        else:
            assert 0 < ray.hit.sum() < 0.9 * (sphere_depth(K, E, 48, 36, R) > 0).sum()


def test_a_step_that_does_not_advance_is_a_miss():
    """a camera 3e6 m away: len + 0.02 == len in float32, so the oracle ends the march as a miss at entry; the float64
    march advances and hits the sphere"""
    vol = written(32, 2.0, 0.125, sphere_sdf(0.6))
    K, E = axis_camera([-3.0e6, 0.0, 0.0], 0, 1)
    assert np.float32(3.0e6) + np.float32(0.02) == np.float32(3.0e6)
    rows = vol.raycast(K, E, 1, 1, 0.04, False)
    r = X.raycast64(vol.tw, vol.col, vol.length, vol.res, vol.origin, vol.ct, K, E, 0.04, 1, 1)
    assert not np.isfinite(rows[0][0, 0]) and r.hit[0]
    assert abs(r.points[0, 0] + 0.6) < 2.0 / 32
