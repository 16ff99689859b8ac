"""CPU: the VoxelGrid operations restatement (oracle/voxelgrid_ops.c) -- the checker of csrc/voxelgrid.cu.

- Numpy restatements of CreateDense, CheckIfIncluded, += / AddVoxels, paint and select.
- Hand-worked answers: a 2x3x4 dense grid, a unit cube carved by one frontal camera, a two-grid merge with
  overlapping colours, an occupancy grid of resolution 8 with three occupied cells.
- Carving against a float64 restatement: every voxel whose decision differs is listed with its margin, which must stay
  within a stated bound.
- The reference's quirks (CarveSilhouette uses the depth test; a uint8 mask is outside everywhere; the zero vector for
  an absent centre) and this project's deviations (non-finite queries, z == 0 and NaN projections, SelectByIndex's
  inverted complement with repeated indices, the OccupancyGrid voxel origin)."""
import numpy as np
import pytest

from cupoch_b200.testing.datagen import sphere_depth
from oracle import voxelgrid_ops_py as V


def frontal_camera(w=64, h=64, f=64.0, dist=3.0):
    """a camera on the -z side of the origin looking along +z: K, 4x4 world-to-camera extrinsic"""
    K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], np.float32)
    E = np.eye(4, dtype=np.float32)
    E[2, 3] = dist
    return K, E


def test_dense_2x3x4_known_answer():
    assert V.dense_counts(0.5, 1.0, 1.5, 2.0) == (2, 3, 4)
    keys, cols = V.create_dense(0.5, 1.0, 1.5, 2.0)
    want = np.array([[x, y, z] for x in range(2) for y in range(3) for z in range(4)], np.int32)
    assert np.array_equal(keys, want) and np.all(cols == 1.0)
    # lexicographic and unique: the reference's sort + unique change nothing
    assert np.array_equal(np.unique(keys, axis=0), keys)


def test_dense_counts_round_in_float_and_reject_bad_arguments():
    # int(std::round(w / vs)): the float32 quotient, rounded half away from zero
    def rnd(w):
        return int(np.floor(np.float64(np.float32(w) / np.float32(0.1)) + 0.5))
    assert V.dense_counts(0.1, 0.25, 0.35, 0.0) == (rnd(0.25), rnd(0.35), 0)
    assert V.dense_counts(0.1, -0.04, 1, 1) == (0, 10, 10)  # rounds to -0
    for bad in [(0.0, 1, 1, 1), (-1.0, 1, 1, 1), (np.nan, 1, 1, 1), (np.inf, 1, 1, 1), (0.1, -1, 1, 1), (0.1, np.nan, 1, 1),
                (0.1, np.inf, 1, 1), (1e-9, 1e3, 1, 1)]:
        assert V.dense_counts(*bad) is None, bad


def test_check_if_included_matches_numpy_and_rejects_non_finite():
    rng = np.random.default_rng(3)
    keys = rng.integers(-20, 20, (3000, 3)).astype(np.int32)
    vs, o = 0.05, np.array([0.1, -0.2, 0.3], np.float32)
    q = (rng.uniform(-1.2, 1.2, (5000, 3)) + o).astype(np.float32)
    q[:5] = [np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [1e30, 0, 0], [0, 0, -1e30]
    got = V.check_if_included(keys, vs, o, q)
    with np.errstate(invalid="ignore"):
        cell = np.floor((q - o) / np.float32(vs))
    finite = np.all(np.isfinite(cell) & (np.abs(cell) < 2 ** 31), 1)
    have = {tuple(k) for k in keys.tolist()}
    want = np.array([bool(f) and tuple(int(x) for x in c) in have for f, c in zip(finite, np.nan_to_num(cell))])
    assert np.array_equal(got, want) and not got[:5].any() and got.sum() > 100
    # unsorted, repeated keys give the same answer
    perm = rng.permutation(np.concatenate([keys, keys[:500]]))
    assert np.array_equal(V.check_if_included(perm, vs, o, q), got)
    assert not V.check_if_included(np.zeros((0, 3), np.int32), vs, o, q).any()


def test_merge_known_answer_and_numpy():
    ka = np.array([[0, 0, 0], [0, 0, 1], [1, 0, 0]], np.int32)
    ca = np.array([[1, 0, 0], [0.2, 0.4, 0.6], [0, 0, 1]], np.float32)
    kb = np.array([[0, 0, 1], [2, 0, 0]], np.int32)
    cb = np.array([[0.6, 0.4, 0.3], [0, 1, 0]], np.float32)
    k, c = V.merge(ka, ca, kb, cb, True)
    assert np.array_equal(k, [[0, 0, 0], [0, 0, 1], [1, 0, 0], [2, 0, 0]])
    assert np.array_equal(c[1], (ca[1] + cb[0]) / np.float32(2)) and np.array_equal(c[[0, 2, 3]], [ca[0], ca[2], cb[1]])
    # AddVoxels keeps the existing voxel of a repeated key
    k2, c2 = V.merge(ka, ca, kb, cb, False)
    assert np.array_equal(k2, k) and np.array_equal(c2[1], ca[1])
    # assigned keys that repeat: the run is summed left to right in the stated order, then divided
    rng = np.random.default_rng(5)
    kk = rng.integers(0, 4, (400, 3)).astype(np.int32)
    cc = rng.random((400, 3)).astype(np.float32)
    k3, c3 = V.merge(kk[:250], cc[:250], kk[250:], cc[250:], True)
    uk = np.unique(kk, axis=0)
    assert np.array_equal(k3, uk)
    for key, col in zip(k3, c3):
        run = cc[np.all(kk == key, 1)]
        s = run[0].copy()
        for r in run[1:]:
            s = (s + r).astype(np.float32)
        assert np.array_equal(col, (s / np.float32(len(run))).astype(np.float32))


def test_paint_and_select():
    keys = np.arange(30, dtype=np.int32).reshape(10, 3)
    cols = np.ones((10, 3), np.float32)
    assert np.array_equal(V.paint(cols, [2, 5], (0, 1, 0))[[2, 5]], [[0, 1, 0]] * 2)
    k, _ = V.select(keys, cols, [7, 1, 7])
    assert np.array_equal(k, keys[[7, 1, 7]])
    # deviation: the inverted selection is the ascending complement of the distinct indices (the reference sizes its
    # output n - len(indices), which is wrong when indices repeat)
    k, _ = V.select(keys, cols, [7, 1, 7], invert=True)
    assert np.array_equal(k, keys[[0, 2, 3, 4, 5, 6, 8, 9]])


def cube_keys(vs):
    """the voxels of the unit cube [-0.5, 0.5]^3 on a grid of voxel size vs whose origin is the cube's corner"""
    n = int(round(1 / vs))
    return V.create_dense(vs, 1, 1, 1)[0], np.full(3, -0.5, np.float32), n


def test_carve_unit_cube_one_frontal_camera():
    """A flat depth map at z = 2.75 in front of the cube (camera at z = -3): the cube spans camera depths 2.5 .. 3.5, so
    a voxel survives when one of its corners has camera depth >= 2.75, i.e. every voxel whose back face is behind the
    plane.  With a pixel-tight image, voxels projecting outside are removed (keep_outside = False) or kept (True)."""
    vs = 0.125
    keys, o, n = cube_keys(vs)
    K, E = frontal_camera()
    depth = np.full((64, 64), 2.75, np.float32)
    keep = V.carve_keep(keys, vs, o, depth, K, E, False)
    back = (keys[:, 2] + 1) * vs - 0.5 + 3.0  # camera depth of the voxel's back corners
    assert np.array_equal(keep, back >= 2.75)
    assert keep.sum() == n * n * 7  # the front layer's back face is at depth 2.625
    # a depth map that sees nothing (0 = invalid) carves everything, unless out-of-image corners keep voxels
    zero = np.zeros((64, 64), np.float32)
    assert not V.carve_keep(keys, vs, o, zero, K, E, False).any()
    # a tiny image: every corner lands outside
    K2 = K.copy()
    K2[0, 2] = K2[1, 2] = 1000.0
    assert V.carve_keep(keys, vs, o, depth, K2, E, True).all()
    assert not V.carve_keep(keys, vs, o, depth, K2, E, False).any()


def test_quirk_silhouette_is_the_depth_test_and_uint8_is_outside():
    vs = 0.25
    keys, o, _ = cube_keys(vs)
    K, E = frontal_camera()
    mask_f = np.ones((64, 64), np.float32)  # a float "mask" of ones acts as depth 1: nothing reaches z >= 1 ... z >= 2.5
    assert V.carve_keep(keys, vs, o, mask_f, K, E, False).all()  # z >= d holds: every voxel survives
    mask_u8 = np.full((64, 64), 255, np.uint8)  # the reference's FloatValueAt refuses any non-float32 image
    assert not V.carve_keep(keys, vs, o, mask_u8, K, E, False).any()
    assert V.carve_keep(keys, vs, o, mask_u8, K, E, True).all()


def nan_camera():
    """fx = fy = 0 with the principal point inside the image: every corner with z != 0 projects to (cx, cy), every
    corner with z == 0 to u = v = 0 / 0 = NaN"""
    K = np.array([[0, 0, 3.5], [0, 0, 2.5], [0, 0, 1]], np.float32)
    return K, np.eye(4, dtype=np.float32)


def test_deviation_z_zero_and_nan_projection_are_outside():
    """Voxel 0 has four corners at z = 0 (u = v = NaN) and four at z = 1; voxel 1 has its corners at z = 1 and 2.  The
    depth 100 everywhere keeps no voxel through the depth test, so only an outside corner can keep one.  Defined here:
    the z = 0 corners are outside, so with keep_voxels_outside_image voxel 0 survives.  Without the guard the NaN would
    pass the bounds test, (int)NaN would clamp into the image and the sample would be NaN: 'inside', failing d > 0,
    and voxel 0 would be removed."""
    K, E = nan_camera()
    keys = np.array([[0, 0, 0], [0, 0, 1]], np.int32)
    img = np.full((6, 8), 100.0, np.float32)
    o = np.zeros(3, np.float32)
    assert V.carve_keep(keys, 1.0, o, img, K, E, True).tolist() == [True, False]
    assert V.carve_keep(keys, 1.0, o, img, K, E, False).tolist() == [False, False]
    # the same corners with a depth they reach (d = 0.5 <= z = 1): both voxels survive through the depth test
    assert V.carve_keep(keys, 1.0, o, np.full((6, 8), 0.5, np.float32), K, E, False).tolist() == [True, True]


def carve_margin64(keys, vs, o, depth, K, E):
    """float64 restatement: per voxel the decision and, over its corners, the smallest |z - d|, |d| (the d > 0 test at
    a silhouette's edge) or distance to the image border: how close the float32 decision was to flipping"""
    h, w = depth.shape
    c = (keys.astype(np.float64) + 0.5) * vs + o.astype(np.float64)
    r = vs / 2
    keep = np.zeros(len(keys), bool)
    margin = np.full(len(keys), np.inf)
    for j in range(8):
        p = c + np.array([(j >> 1) & 1, (j >> 2) & 1, j & 1], np.float64) * 2 * r - r
        x = p @ E[:3, :3].astype(np.float64).T + E[:3, 3].astype(np.float64)
        m = x @ K.astype(np.float64).T
        z = m[:, 2]
        u, v = m[:, 0] / z, m[:, 1] / z
        inside = (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
        ui = np.clip(np.floor(np.where(inside, u, 0)).astype(int), 0, w - 2)
        vi = np.clip(np.floor(np.where(inside, v, 0)).astype(int), 0, h - 2)
        pu, pv = u - ui, v - vi
        d = (depth[vi, ui] * (1 - pv) + depth[vi + 1, ui] * pv) * (1 - pu) + (depth[vi, ui + 1] * (1 - pv) + depth[vi + 1, ui + 1] * pv) * pu
        keep |= inside & (d > 0) & (z >= d)
        border = np.minimum.reduce([np.abs(u), np.abs(u - (w - 1)), np.abs(v), np.abs(v - (h - 1))])
        margin = np.minimum(margin, np.where(inside, np.minimum(np.abs(z - d), np.abs(d)), np.inf))
        margin = np.minimum(margin, border * z / K[0, 0])
    return keep, margin


def test_carve_against_float64_restatement():
    """A sphere's depth map seen from an oblique camera.  Decisions that differ between float32 and float64 are listed
    with their margins; each must be within 1e-5 (a few float32 ulps of the depths and coordinates used)."""
    vs = 1 / 64
    keys = V.create_dense(vs, 2, 2, 2)[0]
    o = np.full(3, -1.0, np.float32)
    K, E = frontal_camera(96, 96, 80.0, 4.0)
    ang = 0.3
    R = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    E[:3, :3] = R
    E[:3, 3] = [0, 0, 4.0]
    depth = sphere_depth(K, E, 96, 96, 0.7)
    got = V.carve_keep(keys, vs, o, depth, K, E, False)
    ref, margin = carve_margin64(keys, vs, o, depth, K, E)
    diff = np.flatnonzero(got != ref)
    listed = [(int(i), float(margin[i])) for i in diff]
    assert got.sum() > 1000 and len(diff) <= 0.001 * len(keys), listed[:20]
    assert all(m <= 1e-5 for _, m in listed), listed[:20]


def test_occupancy_grid_resolution_8_three_cells():
    cells = np.array([[0, 0, 0], [3, 4, 5], [7, 7, 7]], np.int32)
    vs, o, res = 0.5, np.array([1, 2, 3], np.float32), 8
    pts = V.occ_points(cells, res, vs, o)
    assert np.array_equal(pts, (cells - 4 + 0.5) * 0.5 + o)  # exact in binary
    vo = V.occ_voxel_origin(res, vs, o)
    assert np.array_equal(vo, o - 2.0)
    # deviation: the voxel centre of each cell is its point (the reference keeps the grid origin: 4 cells off)
    assert np.array_equal((cells + 0.5) * vs + vo, pts)
    assert np.all(np.abs((cells + 0.5) * vs + o - pts) == 2.0)
