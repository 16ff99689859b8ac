"""OccupancyGrid::Insert on the device against the float64 model of cupoch_b200/testing/occgrid64.py (and bit for bit
against the CPU oracle, which walks with the same rule): random rays in all octants, exact known answers at ties and
faces, rays outside the grid, max_range, far origins, long rays, clamping across calls, ray counts around the block
and warp sizes, small, odd and the largest resolutions, and a 1 M-ray fan into 512^3."""
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cupoch_b200 as cph
from cupoch_b200.testing import occgrid64 as M

G = cph.geometry
ORG = (0.1, -0.2, 0.05)


def _dense(g):
    return g.to_torch().cpu().numpy().reshape(-1).copy()


def _bounds(g):
    lo, hi = g._bounds()
    return np.concatenate([lo, hi]).astype(np.int64)


def _insert(g, o, pts, vp, max_range=-1.0, full=True, label=""):
    """one Insert on the device grid g (and on the oracle grid o, if given): the device against the model, and against
    the oracle bit for bit (the dense array and the bounds) -> the model's info"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    p0, b0 = _dense(g), _bounds(g)
    g.insert(G.PointCloud(pts), vp, max_range)
    p1, b1 = _dense(g), _bounds(g)
    if o is not None:
        o.insert(pts, vp, max_range)
        np.testing.assert_array_equal(p1.view(np.uint32), o.prob.view(np.uint32), err_msg=label)
        np.testing.assert_array_equal(b1, o.bounds.astype(np.int64), err_msg=label)
    return M.check_insert(p0, p1, b0, b1, pts, vp, g.origin, g.voxel_size, g.resolution, max_range,
                          params=(g.clamping_thres_min, g.clamping_thres_max, g.prob_hit_log, g.prob_miss_log),
                          full=full, label=label)


def _fan(rng, n, vp, r0, r1):
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (np.float32(vp) + d * rng.uniform(r0, r1, (n, 1))).astype(np.float32)


def _pair(orc, vs, res, org):
    return G.OccupancyGrid(vs, res, org), orc.OccupancyGrid(vs, res, org)


@pytest.mark.parametrize("vs", [0.05, 1.0])
def test_random_rays_all_octants(orc, vs):
    rng = np.random.default_rng(41)
    g, o = _pair(orc, vs, 160, ORG)
    for k in range(3):
        vp = (rng.uniform(-20, 20, 3) * vs).astype(np.float32)
        _insert(g, o, _fan(rng, 5000, vp, 0.5 * vs, 60 * vs), vp, label="vs %g call %d" % (vs, k))


def test_axis_aligned_rays_both_directions(orc):
    g, o = _pair(orc, 0.05, 160, ORG)
    vp = np.float32([0.013, 0.027, -0.011])
    pts = []
    for a in range(3):
        for sgn in (1, -1):
            for r in (0.33, 1.01, 2.5, 3.77):
                p = vp.copy()
                p[a] += sgn * r
                pts.append(p)
    _insert(g, o, np.array(pts), vp, label="axis aligned")


@pytest.mark.parametrize("case", M.KNOWN_ANSWERS, ids=[k[0] for k in M.KNOWN_ANSWERS])
def test_exact_known_answers(case):
    name, start, end, free, occ = case
    h = 32
    g = G.OccupancyGrid(0.25, 64, (0, 0, 0))
    _insert(g, None, [end], start, label=name)
    idx, _ = g.extract_free_voxels()
    assert {tuple(v) for v in idx.tolist()} == {(x + h, y + h, z + h) for x, y, z in free}
    idx, _ = g.extract_occupied_voxels()
    assert {tuple(v) for v in idx.tolist()} == {(occ[0] + h, occ[1] + h, occ[2] + h)}


def test_reference_rule_hand_worked_ray():
    """the ray of test_oracle_occgrid64::test_reference_rule_hand_worked_ray: the device marks the cells the segment
    crosses, (2,0) included and (1,1) not"""
    g = G.OccupancyGrid(1.0, 8, (0, 0, 0))
    g.insert(np.float32([[3.75, 1.25, 0.5]]), (0.25, 0.25, 0.5))
    idx, _ = g.extract_free_voxels()
    assert {tuple(v) for v in idx.tolist()} == {(4, 4, 4), (5, 4, 4), (6, 4, 4), (6, 5, 4)}


def test_outside_leave_reenter_and_entirely_outside(orc):
    rng = np.random.default_rng(42)
    g, o = _pair(orc, 0.05, 64, (0, 0, 0))
    vp = np.float32([2.5, -2.1, 0.3])
    _insert(g, o, _fan(rng, 3000, vp, 1.0, 6.0), vp, label="viewpoint outside")
    vp = np.float32([0.0, 0.0, 0.0])
    _insert(g, o, _fan(rng, 3000, vp, 1.0, 4.0), vp, label="rays that leave")
    a = np.float32([-2.0, -1.9, 0.1])
    _insert(g, o, (np.float32([2.0, 1.7, -0.1]) + rng.uniform(-0.3, 0.3, (800, 3))).astype(np.float32), a,
            label="chords through the grid")
    before = _dense(g)
    far = np.float32([10.0, 10.0, 10.0])
    _insert(g, o, _fan(rng, 800, far, 0.5, 3.0), far, label="entirely outside")
    assert (_dense(g).view(np.uint32) == before.view(np.uint32)).all()


def test_max_range(orc):
    rng = np.random.default_rng(43)
    for mr in (-1.0, 1.5, 3.0, 0.0):
        g, o = _pair(orc, 0.05, 160, ORG)
        vp = np.float32([0.3, -0.1, 0.2])
        pts = _fan(rng, 5000, vp, 0.2, 4.5)
        pts[:4] = vp                                          # zero-length rays: hits, never cut
        info = _insert(g, o, pts, vp, mr, label="max_range %g" % mr)
        assert info["cut_disagree"] == 0
    vs, h = 0.25, 32
    vp = np.float32([0.125, 0.125, 0.125])
    g = G.OccupancyGrid(vs, 64, (0, 0, 0))
    _insert(g, None, np.float32([[0.875, 1.125, 0.125]]), vp, 1.25, label="dist == max_range")   # 3-4-5: exact
    assert {tuple(v) for v in g.extract_occupied_voxels()[0].tolist()} == {(3 + h, 4 + h, h)}
    g = G.OccupancyGrid(vs, 64, (0, 0, 0))
    _insert(g, None, np.float32([[2.125, 0.125, 0.125]]), vp, 1.0, label="cut")
    assert len(g.extract_occupied_voxels()[1]) == 0
    assert {tuple(v) for v in g.extract_free_voxels()[0].tolist()} == {(x + h, h, h) for x in range(4)}
    g = G.OccupancyGrid(vs, 64, (0, 0, 0))
    _insert(g, None, np.float32([[2.125, 0.125, 0.125]]), vp, 0.0, label="cut to zero length")
    assert np.isnan(_dense(g)).all()


def test_far_origins_negative_grid_coordinates(orc):
    rng = np.random.default_rng(44)
    for org in ((1000.0, -1000.0, 1000.0), (-1000.0, 1000.0, -1000.0)):
        g, o = _pair(orc, 0.05, 160, org)
        vp = (np.float32(org) + np.float32([-0.5, 0.3, -1.0])).astype(np.float32)
        info = _insert(g, o, _fan(rng, 5000, vp, 0.3, 4.5), vp, label="origin %r" % (org,))
        assert info["free"] > 0


def test_long_rays_and_the_ray_that_sets_n_div(orc):
    rng = np.random.default_rng(45)
    g, o = _pair(orc, 0.05, 512, (0, 0, 0))
    vp = np.float32([0.013, -0.021, 0.007])
    pts = _fan(rng, 2000, vp, 5.0, 12.0)
    pts[0] = vp + np.float32([12.0, 11.5, -11.75])            # the L_inf ray sets n_div
    pts[1] = vp + np.float32([-12.0, -12.0, 12.0])
    info = _insert(g, o, pts, vp, label="long")
    assert info["required"] > 2000 * 100
    g, o = _pair(orc, 0.5, 256, (3000.0, -3000.0, 2000.0))
    vp = (np.float32([3000.1, -2999.8, 2000.3])).astype(np.float32)
    steps = rng.integers(-100, 101, (500, 3)).astype(np.float32)
    steps[:, 0] = np.where(np.abs(steps[:, 0]) < 1, 100, steps[:, 0])
    _insert(g, o, (vp + steps * np.float32(0.5)).astype(np.float32), vp, label="3 km, integer-voxel extents")


def test_successive_inserts_reach_both_clamps(orc):
    rng = np.random.default_rng(46)
    vs = 0.1
    g, o = _pair(orc, vs, 64, (0, 0, 0))
    wall = np.stack(np.meshgrid(np.linspace(-1.0, 1.0, 40), np.linspace(-1.0, 1.0, 40), indexing="ij"), -1).reshape(-1, 2)
    front = np.concatenate([wall, np.full((len(wall), 1), 1.23)], 1).astype(np.float32)
    back = np.concatenate([wall, np.full((len(wall), 1), 2.27)], 1).astype(np.float32)
    vp = np.float32([0.03, 0.02, -1.0])
    for k in range(8):
        pts = (front if k % 2 == 0 else back) + rng.uniform(-0.004, 0.004, front.shape).astype(np.float32)
        _insert(g, o, pts, vp, label="call %d" % k)
    p = _dense(g)
    assert (p == np.float32(g.clamping_thres_min)).any()
    g, o = _pair(orc, vs, 64, (0, 0, 0))
    cell = o.voxel_index([0.0, 0.0, 1.23])
    for k in range(6):
        _insert(g, o, front, vp, label="front %d" % k)
    assert _dense(g)[cell] == np.float32(g.clamping_thres_max)
    _insert(g, o, back, vp, label="freed after the clamp")   # occupied in the last call, free in this one
    assert _dense(g)[cell] == np.float32(np.float32(g.clamping_thres_max) + np.float32(g.prob_miss_log))


@pytest.mark.parametrize("n", [1, 31, 32, 33, 127, 128, 129])
def test_ray_counts_and_bounds(orc, n):
    """n around the 128-thread traversal blocks and the warp reductions of the bounds; the bounds after every call"""
    rng = np.random.default_rng(47 + n)
    g, o = _pair(orc, 0.05, 160, ORG)
    for k in range(3):
        vp = rng.uniform(-0.5, 0.5, 3).astype(np.float32)
        _insert(g, o, _fan(rng, n, vp, 0.1, 3.0), vp, label="n %d call %d" % (n, k))


@pytest.mark.parametrize("res", [2, 63, 65])
def test_small_and_odd_resolutions(orc, res):
    rng = np.random.default_rng(48 + res)
    vs = 0.1
    g, o = _pair(orc, vs, res, (0.01, -0.02, 0.03))
    vp = np.float32([0.011, 0.004, -0.013])
    for k in range(2):
        _insert(g, o, _fan(rng, 2000, vp, 0.05, res * vs * 0.8), vp, label="res %d call %d" % (res, k))


def test_set_free_area_and_point_queries_near_faces():
    vs, res, h = 0.25, 64, 32
    g = G.OccupancyGrid(vs, res, (0, 0, 0))
    lo_b, hi_b = (0.25, -0.25, 0.0), (0.5, 0.2, 0.7)
    g.set_free_area(lo_b, hi_b)
    lo, hi = M.free_area_box(lo_b, hi_b, (0, 0, 0), vs, res)
    np.testing.assert_array_equal(_bounds(g), np.concatenate([lo, hi]))
    p = _dense(g).reshape(res, res, res)
    box = np.zeros((res,) * 3, bool)
    box[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = True
    assert (p[box] == np.float32(g.prob_miss_log)).all() and np.isnan(p[~box]).all()
    for q in ((0.25, 0.0, 0.0), (0.25 - 2 ** -10, 0.0, 0.0), (-0.25, 0.0, 0.0), (-0.25 - 2 ** -10, -2 ** -12, 0.5),
              (0.5, 0.25, 0.75), (100.0, 0.0, 0.0), (-8.0, -8.0, -8.0), (7.99, 7.99, 7.99), (8.0, 0.0, 0.0)):
        i = M.voxel_index(q, (0, 0, 0), vs, res)
        want = i >= 0 and bool(box.reshape(-1)[i])
        assert g.get_voxel(q)[0] == want and g.is_unknown(q) == (not want), q
        assert not g.is_occupied(q)


def test_largest_resolution_last_cell():
    """res 1290: one ray ends in cell (1289, 1289, 1289), linear index 1290^3 - 1, the largest that fits an int.  The
    ray crosses 1,933 cells; at this length the model's worst-case delta is 0.3 vs, so 644 of them are required"""
    import torch
    res, vs = 1290, 1.0
    h = res // 2
    g = G.OccupancyGrid(vs, res, (0, 0, 0))
    vp = np.float32([0.37, 0.21, 0.13])
    end = np.float32([[644.6, 644.7, 644.55]])
    g.insert(G.PointCloud(end), vp)
    t = g.to_torch().reshape(-1)
    assert float(t[res ** 3 - 1]) == np.float32(g.prob_hit_log)
    R = M.form_rays(end, vp, (0, 0, 0))
    req, alw = M.ray_sets(R["s"], R["e"][0], vs)
    req = np.array(sorted(req), np.int64).reshape(-1, 3) + h
    assert len(req) > 500
    v = t[torch.as_tensor((req[:, 0] * res + req[:, 1]) * res + req[:, 2], device=t.device)].cpu().numpy()
    assert (v == np.float32(g.prob_miss_log)).all()
    known = torch.nonzero(~torch.isnan(t)).reshape(-1).cpu().numpy()
    kn = np.stack(np.unravel_index(known, (res,) * 3), 1)
    assert {tuple(x) for x in kn.tolist()} <= {(x + h, y + h, z + h) for x, y, z in alw} | {(res - 1,) * 3}
    lo, hi = g._bounds()
    assert hi.tolist() == [res - 1] * 3 and lo.tolist() == kn.min(0).tolist()
    del t, g
    gc.collect()
    torch.cuda.synchronize()


def test_million_ray_fan_512(orc):
    """1 M rays into 512^3: bit parity with the oracle; the model's required cells on a 50 k-ray subset (a union over
    rays, so a subset checks only that its required cells are freed)"""
    rng = np.random.default_rng(49)
    g, o = _pair(orc, 0.05, 512, (0, 0, 0))
    vp = np.float32([0.013, -0.007, 0.021])
    pts = _fan(rng, 1_000_000, vp, 2.0, 10.0)
    p0, b0 = _dense(g), _bounds(g)
    g.insert(G.PointCloud(pts), vp)
    o.insert(pts, vp)
    p1, b1 = _dense(g), _bounds(g)
    np.testing.assert_array_equal(p1.view(np.uint32), o.prob.view(np.uint32))
    np.testing.assert_array_equal(b1, o.bounds.astype(np.int64))
    del o
    gc.collect()
    sub = rng.choice(len(pts), 50_000, replace=False)
    info = M.check_insert(p0, p1, b0, b1, pts[sub], vp, g.origin, g.voxel_size, g.resolution, full=False,
                          label="1 M fan, 50 k subset")
    assert info["required"] > 50_000 * 50
