"""The OccupancyGrid restatement (oracle/oracle.c) against the float64 model of cupoch_b200/testing/occgrid64.py: the
library's ray walk passes it on every family, the reference's half-voxel boundary fails it on nearly every ray, and
hand-worked rays pin the cells both rules mark."""
import contextlib
import io

import numpy as np
import pytest

from cupoch_b200.testing import occgrid64 as M
from oracle import oracle_py as orc

ORG = (0.1, -0.2, 0.05)


def _insert(g, pts, vp, max_range=-1.0, ref_rule=False, full=True, label=""):
    """one Insert on the oracle grid g, checked against the model -> the model's info"""
    p0, b0 = g.prob.copy(), g.bounds.copy()
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    g.insert(pts, vp, max_range, ref_rule=ref_rule)
    return M.check_insert(p0, g.prob, b0, g.bounds, pts, vp, g.origin, g.voxel_size, g.resolution, max_range,
                          params=(g.clamping_thres_min, g.clamping_thres_max, g.prob_hit_log, g.prob_miss_log),
                          full=full, label=label)


def _fan(rng, n, vp, r0, r1):
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (np.float32(vp) + d * rng.uniform(r0, r1, (n, 1))).astype(np.float32)


def _free_cells(g):
    idx, pr = g.extract(1)
    return {tuple(v) for v in idx.tolist()}


@pytest.mark.parametrize("vs", [0.05, 1.0])
def test_random_rays_all_octants(vs):
    rng = np.random.default_rng(21)
    g = orc.OccupancyGrid(vs, 160, ORG)
    for k in range(3):
        vp = (rng.uniform(-20, 20, 3) * vs).astype(np.float32)
        _insert(g, _fan(rng, 3000, vp, 0.5 * vs, 60 * vs), vp, label="vs %g call %d" % (vs, k))


@pytest.mark.parametrize("vs", [0.05, 1.0])
def test_reference_rule_fails_the_model_on_nearly_every_ray(vs):
    """one ray per Insert: the library's walk passes every ray, the reference's (cur + 0.5 step) vs fails nearly all"""
    rng = np.random.default_rng(22)
    bad = {False: 0, True: 0}
    for i in range(150):
        vp = (rng.uniform(-30, 30, 3) * vs).astype(np.float32)
        p = _fan(rng, 1, vp, 2 * vs, 40 * vs)
        for ref in (False, True):
            g = orc.OccupancyGrid(vs, 160, ORG)
            try:
                with contextlib.redirect_stdout(io.StringIO()):
                    _insert(g, p, vp, ref_rule=ref)
            except AssertionError:
                bad[ref] += 1
    print("rays failing the model of 150: library rule %d, reference rule %d" % (bad[False], bad[True]))
    assert bad[False] == 0
    assert bad[True] >= 140


def test_reference_rule_hand_worked_ray():
    """vs 1, start (0.25, 0.25, 0.5), end (3.75, 1.25, 0.5): the segment crosses x = 1, 2 at y < 1 and y = 1 at x = 2.875,
    so it passes through cells (0,0) (1,0) (2,0) (2,1) and ends in (3,1).  The reference's first boundaries are x = 0.5,
    y = 0.5: it crosses y at x = 1.125, marks (1,1), which the segment never enters, and misses (2,0)."""
    h = 4
    start, end = (0.25, 0.25, 0.5), (3.75, 1.25, 0.5)
    want = {(0, 0), (1, 0), (2, 0), (2, 1)}
    ref = {(0, 0), (1, 0), (1, 1), (2, 1)}
    for rule, cells in ((False, want), (True, ref)):
        g = orc.OccupancyGrid(1.0, 8, (0, 0, 0))
        g.insert([end], start, ref_rule=rule)
        assert _free_cells(g) == {(x + h, y + h, h) for x, y in cells}
        assert {tuple(v) for v in g.extract(2)[0].tolist()} == {(3 + h, 1 + h, h)}
    req, alw = M.ray_sets(np.float64(start), np.float64(end), 1.0)
    assert {(x, y, 0) for x, y in want} == req
    assert (1, 1, 0) not in alw and (2, 0, 0) in req


@pytest.mark.parametrize("case", M.KNOWN_ANSWERS, ids=[k[0] for k in M.KNOWN_ANSWERS])
def test_exact_known_answers(case):
    name, start, end, free, occ = case
    h = 32
    g = orc.OccupancyGrid(0.25, 64, (0, 0, 0))
    _insert(g, [end], start, label=name)
    assert _free_cells(g) == {(x + h, y + h, z + h) for x, y, z in free}
    assert {tuple(v) for v in g.extract(2)[0].tolist()} == {(occ[0] + h, occ[1] + h, occ[2] + h)}
    req, alw = M.ray_sets(np.float64(start), np.float64(end), 0.25)
    assert req - {occ} <= set(free) <= alw                   # occupied beats free


def test_max_range_cut_equal_and_zero_length():
    """max_range < 0: no cut; a cut ray frees up to the cut and its end cell stays unknown; dist == max_range is a hit;
    zero-length rays change nothing, cut or not"""
    vs, h = 0.25, 32
    vp = np.float32([0.125, 0.125, 0.125])
    far = np.float32([[2.125, 0.125, 0.125]])
    g = orc.OccupancyGrid(vs, 64, (0, 0, 0))
    _insert(g, far, vp, -1.0, label="no cut")
    assert {tuple(v) for v in g.extract(2)[0].tolist()} == {(8 + h, h, h)}
    g = orc.OccupancyGrid(vs, 64, (0, 0, 0))
    _insert(g, far, vp, 1.0, label="cut")                 # ranged = 1.125: cell 4, neither free nor occupied
    assert len(g.extract(2)[0]) == 0
    assert _free_cells(g) == {(x + h, h, h) for x in range(4)}
    g = orc.OccupancyGrid(vs, 64, (0, 0, 0))
    p = np.float32([[0.125 + 0.75, 0.125 + 1.0, 0.125]])   # a 3-4-5 triangle: dist == 1.25 exactly
    _insert(g, p, vp, 1.25, label="equal")
    assert {tuple(v) for v in g.extract(2)[0].tolist()} == {(3 + h, 4 + h, h)}
    for mr in (-1.0, 0.5, 0.0):
        g = orc.OccupancyGrid(vs, 64, (0, 0, 0))
        _insert(g, np.repeat(vp[None], 3, 0), vp, mr, label="zero length %g" % mr)
        assert len(_free_cells(g)) == 0
        assert len(g.extract(2)[0]) == 1                    # dist 0 <= max_range: a hit
    g = orc.OccupancyGrid(vs, 64, (0, 0, 0))
    _insert(g, far, vp, 0.0, label="cut to zero length")    # ranged = the viewpoint: no cell changes
    assert np.isnan(g.prob).all()


@pytest.mark.parametrize("mr", [-1.0, 1.5, 3.0])
def test_random_rays_with_max_range(mr):
    rng = np.random.default_rng(23)
    g = orc.OccupancyGrid(0.05, 160, ORG)
    vp = np.float32([0.3, -0.1, 0.2])
    pts = _fan(rng, 4000, vp, 0.2, 4.5)
    pts[:4] = vp
    info = _insert(g, pts, vp, mr, label="max_range %g" % mr)
    assert info["cut_disagree"] == 0


def test_outside_the_grid_leave_reenter_and_entirely_outside():
    rng = np.random.default_rng(24)
    vs, res = 0.05, 64
    g = orc.OccupancyGrid(vs, res, (0, 0, 0))
    vp = np.float32([2.5, -2.1, 0.3])                     # outside the 3.2 m grid
    _insert(g, _fan(rng, 2000, vp, 1.0, 6.0), vp, label="viewpoint outside")
    vp = np.float32([0.0, 0.0, 0.0])                       # from inside, out through a side
    _insert(g, _fan(rng, 2000, vp, 1.0, 4.0), vp, label="rays that leave")
    # chords from outside to outside: they enter and leave the grid (a segment meets the box once), end cells outside
    a = np.float32([-2.0, -1.9, 0.1]) + rng.uniform(-0.3, 0.3, (500, 3)).astype(np.float32)
    _insert(g, (np.float32([2.0, 1.7, -0.1]) + rng.uniform(-0.3, 0.3, (500, 3))).astype(np.float32), a[0], label="chords")
    before = g.prob.copy()
    far = np.float32([10.0, 10.0, 10.0])
    _insert(g, _fan(rng, 500, far, 0.5, 3.0), far, label="entirely outside")
    assert (g.prob.view(np.uint32) == before.view(np.uint32)).all()


def test_far_origins_and_negative_grid_coordinates():
    rng = np.random.default_rng(25)
    for org in ((1000.0, -1000.0, 1000.0), (-1000.0, 1000.0, -1000.0)):
        g = orc.OccupancyGrid(0.05, 160, org)
        vp = (np.float32(org) + np.float32([-0.5, 0.3, -1.0])).astype(np.float32)   # below the grid centre
        info = _insert(g, _fan(rng, 3000, vp, 0.3, 4.5), vp, label="origin %r" % (org,))
        assert info["free"] > 0


def test_long_rays_and_the_ray_that_sets_n_div():
    """rays of hundreds of voxels; the longest ray's L_inf sets n_div, so its walk runs against the 3 (n_div + 1) cap"""
    rng = np.random.default_rng(26)
    vs = 0.05
    g = orc.OccupancyGrid(vs, 512, (0, 0, 0))
    vp = np.float32([0.013, -0.021, 0.007])
    pts = _fan(rng, 500, vp, 5.0, 12.0)
    pts[0] = vp + np.float32([12.0, 11.5, -11.75])          # the L_inf ray, an integer number of voxels per axis
    pts[1] = vp + np.float32([-12.0, -12.0, 12.0])
    info = _insert(g, pts, vp, label="long")
    assert info["required"] > 500 * 100


def test_far_origin_long_rays_integer_voxel_extent():
    """rays whose L_inf is an integer number of voxels on every axis, 3 km from the origin: the cap never truncates"""
    rng = np.random.default_rng(27)
    vs = 0.5
    org = (3000.0, -3000.0, 2000.0)
    g = orc.OccupancyGrid(vs, 256, org)
    vp = (np.float32(org) + np.float32([0.1, 0.2, 0.3])).astype(np.float32)
    steps = rng.integers(-100, 101, (300, 3)).astype(np.float32)
    steps[:, 0] = np.where(np.abs(steps[:, 0]) < 1, 100, steps[:, 0])
    _insert(g, (vp + steps * np.float32(vs)).astype(np.float32), vp, label="3 km")


def test_successive_inserts_reach_both_clamps():
    """eight calls from alternating viewpoints: cells saturate at both clamps, and a cell occupied in one call is freed
    in the next"""
    rng = np.random.default_rng(28)
    vs = 0.1
    g = orc.OccupancyGrid(vs, 64, (0, 0, 0))
    wall = np.stack(np.meshgrid(np.linspace(-1.0, 1.0, 40), np.linspace(-1.0, 1.0, 40), indexing="ij"), -1).reshape(-1, 2)
    front = np.concatenate([wall, np.full((len(wall), 1), 1.23)], 1).astype(np.float32)
    back = np.concatenate([wall, np.full((len(wall), 1), 2.27)], 1).astype(np.float32)
    vp = np.float32([0.03, 0.02, -1.0])
    cell = orc.OccupancyGrid(vs, 64, (0, 0, 0)).voxel_index([0.0, 0.0, 1.23])
    for k in range(8):
        pts = front if k % 2 == 0 else back             # the back wall's rays pass through the front wall's cells
        _insert(g, pts + rng.uniform(-0.004, 0.004, pts.shape).astype(np.float32), vp, label="call %d" % k)
    p = g.prob[~np.isnan(g.prob)]
    assert (p == np.float32(g.clamping_thres_min)).any()
    g2 = orc.OccupancyGrid(vs, 64, (0, 0, 0))
    for k in range(6):
        _insert(g2, front, vp, label="front %d" % k)
    assert g2.prob[cell] == np.float32(g2.clamping_thres_max)
    _insert(g2, back, vp, label="freed after the clamp")
    assert g2.prob[cell] == np.float32(np.float32(g2.clamping_thres_max) + np.float32(g2.prob_miss_log))


@pytest.mark.parametrize("n", [1, 31, 32, 33, 127, 128, 129])
def test_ray_counts(n):
    rng = np.random.default_rng(29 + n)
    g = orc.OccupancyGrid(0.05, 160, ORG)
    for k in range(2):
        vp = rng.uniform(-0.5, 0.5, 3).astype(np.float32)
        _insert(g, _fan(rng, n, vp, 0.1, 3.0), vp, label="n %d call %d" % (n, k))


@pytest.mark.parametrize("res", [2, 63, 65])
def test_small_and_odd_resolutions(res):
    rng = np.random.default_rng(30 + res)
    vs = 0.1
    g = orc.OccupancyGrid(vs, res, (0.01, -0.02, 0.03))
    vp = np.float32([0.011, 0.004, -0.013])
    _insert(g, _fan(rng, 1000, vp, 0.05, res * vs * 0.8), vp, label="res %d" % res)


def test_set_free_area_and_point_queries_near_faces():
    vs, res, h = 0.25, 64, 32
    g = orc.OccupancyGrid(vs, res, (0, 0, 0))
    lo_b, hi_b = (0.25, -0.25, 0.0), (0.5, 0.2, 0.7)      # faces, a negative face, interior points
    g.set_free_area(lo_b, hi_b)
    lo, hi = M.free_area_box(lo_b, hi_b, (0, 0, 0), vs, res)
    assert lo.tolist() == [1 + h, -1 + h, h] and hi.tolist() == [2 + h, h, 2 + h]
    np.testing.assert_array_equal(g.bounds.astype(np.int64), np.concatenate([lo, hi]))
    box = {(x, y, z) for x in range(lo[0], hi[0] + 1) for y in range(lo[1], hi[1] + 1) for z in range(lo[2], hi[2] + 1)}
    assert _free_cells(g) == {(0, 0, 0)} and len(g.extract(1)[0]) == len(box)   # grid_index_ is never written here
    for p in ((0.25, 0.0, 0.0), (0.25 - 2 ** -10, 0.0, 0.0), (-0.25, 0.0, 0.0), (-0.25 - 2 ** -10, -2 ** -12, 0.5),
              (0.5, 0.25, 0.75), (100.0, 0.0, 0.0), (-8.0, -8.0, -8.0), (7.99, 7.99, 7.99), (8.0, 0.0, 0.0)):
        i = M.voxel_index(p, (0, 0, 0), vs, res)
        assert g.voxel_index(p) == i
        known, val = g.get_voxel(p)
        want = i >= 0 and tuple(np.unravel_index(i, (res,) * 3)) in box
        assert known == want, p
