"""GPU: the VoxelGrid operations of csrc/voxelgrid.cu through cph.geometry, against oracle/voxelgrid_ops.c bit for bit.

- CreateDense up to 256^3 (and 512^3 on properties only); CheckIfIncluded of 1 M queries with NaN / inf rows against
  the config-3 cloud voxelised at 0.02 (about 2 M voxels), sorted and after a shuffling select_by_index; += and
  add_voxels of two overlapping 2 M-voxel grids; paint, select and invert on them; carving dense 128^3 and 256^3 grids
  by 8 and 16 views with a depth map and a uint8 mask, both keep_voxels_outside_image values; both
  CreateFromOccupancyGrid calls on a 512^3 grid after a 1 M-ray insert, whose voxels collide with every occupied cell.
- A fixed launch count per call, bit-identical repeats, and the argument rules."""
import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing import datagen
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import voxelgrid_ops_py as V

G, CAM = cph.geometry, cph.camera


def same(vg, keys, cols):
    k, c = vg.get_voxels()
    assert k.shape == keys.shape and np.array_equal(k, keys)
    assert c.shape == cols.shape and np.array_equal(c.view(np.uint32), np.asarray(cols, np.float32).view(np.uint32))


@pytest.mark.parametrize("args", [(0.5, 1.0, 1.5, 2.0), (0.1, 0.25, 0.35, 0.45), (1 / 64, 1, 1, 1), (1 / 256, 1, 1, 1),
                                  (0.1, 0.0, 1.0, 1.0)])
def test_create_dense_matches_oracle(args):
    vs, w, h, d = args
    g = G.VoxelGrid.create_dense((0.1, 0.2, 0.3), vs, w, h, d)
    same(g, *V.create_dense(vs, w, h, d))
    assert g.voxel_size == float(np.float32(vs)) and np.array_equal(g.origin, np.float32([0.1, 0.2, 0.3]))


def test_create_dense_512_properties():
    g = G.VoxelGrid.create_dense((0, 0, 0), 1 / 512, 1, 1, 1)
    assert len(g) == 512 ** 3
    k = g.voxels_keys
    first = np.zeros((1, 3), np.int32)
    last = np.zeros((1, 3), np.int32)
    _lib.check(_lib.lib().cphb_memcpy_d2h(first.ctypes.data, k.ptr, 12, None))
    _lib.check(_lib.lib().cphb_memcpy_d2h(last.ctypes.data, k.ptr + 12 * (len(g) - 1), 12, None))
    assert first.tolist() == [[0, 0, 0]] and last.tolist() == [[511, 511, 511]]
    # lexicographic order: the packed keys of the whole grid are 0, 1, 2, ...
    keys = k.cpu()
    step = 1 << 24
    for s0 in range(0, len(keys), step):
        i = np.arange(s0, s0 + step, dtype=np.int32)
        assert np.array_equal(keys[s0:s0 + step], np.stack([i >> 18, (i >> 9) & 511, i & 511], 1))


@pytest.mark.parametrize("bad", [(0.0, 1, 1, 1), (np.nan, 1, 1, 1), (-0.1, 1, 1, 1), (0.1, -1, 1, 1), (0.1, np.inf, 1, 1),
                                 (1e-9, 1e3, 1e3, 1e3), (1.0, 2e9, 2e9, 2e9)])
def test_create_dense_rejects(bad):
    with pytest.raises(_lib.CphbError):
        G.VoxelGrid.create_dense((0, 0, 0), *bad)


@pytest.fixture(scope="module")
def config3():
    """the config-3 cloud (uniform_cube(10 M, 21) in [0,4)x[0,4)x[0,1)) voxelised at 0.02, with colours, and a second
    grid on the same origin from a shifted cloud that overlaps half of it"""
    pts = datagen.uniform_cube(10_000_000, 21, hi=(4, 4, 1))
    rng = np.random.default_rng(7)
    pc = G.PointCloud(pts)
    pc.colors = rng.random((len(pts), 3)).astype(np.float32)
    lo, hi = np.zeros(3, np.float32), np.float32([6, 4, 1])
    a = G.VoxelGrid.create_from_point_cloud_within_bounds(pc, 0.02, lo, hi)
    pc2 = G.PointCloud((pts + np.float32([2, 0, 0])).astype(np.float32))
    pc2.colors = rng.random((len(pts), 3)).astype(np.float32)
    b = G.VoxelGrid.create_from_point_cloud_within_bounds(pc2, 0.02, lo, hi)
    return a, b


def queries(n, seed):
    rng = np.random.default_rng(seed)
    q = rng.uniform((-0.1, -0.1, -0.1), (4.1, 4.1, 1.1), (n, 3)).astype(np.float32)
    bad = rng.choice(n, 3000, replace=False)
    q[bad[:1000], 0] = np.nan
    q[bad[1000:2000], 1] = np.inf
    q[bad[2000:], 2] = -np.inf
    return q


def test_check_if_included_sorted_and_shuffled(config3):
    a, _ = config3
    assert 1_500_000 < len(a) < 2_500_000
    q = queries(1_000_000, 1)
    keys = a.get_voxels()[0]
    want = V.check_if_included(keys, a.voxel_size, a.origin, q)
    got = a.check_if_included(q)
    assert got.dtype == bool and np.array_equal(got, want) and 0.3 < want.mean() < 0.99
    perm = np.random.default_rng(2).permutation(len(a))
    shuffled = a.select_by_index(perm)
    assert np.array_equal(shuffled.get_voxels()[0], keys[perm])
    assert np.array_equal(shuffled.check_if_included(q), want)
    # repeated keys as well
    rep = a.select_by_index(np.concatenate([perm[:1000], perm]))
    assert np.array_equal(rep.check_if_included(q), want)


def test_voxel_center_and_bounding_points(config3):
    a, _ = config3
    k = a.get_voxels()[0][12345]
    c = a.get_voxel_center_coordinate(k)
    assert np.array_equal(c, (k.astype(np.float32) + np.float32(0.5)) * np.float32(a.voxel_size) + a.origin)
    # the reference's quirk: an absent key gives the zero vector
    assert np.array_equal(a.get_voxel_center_coordinate((-5, -5, -5)), np.zeros(3, np.float32))
    bp = a.get_voxel_bounding_points(k)
    r = np.float32(a.voxel_size) * np.float32(0.5)
    assert bp.shape == (8, 3) and np.array_equal(bp[0], c - r) and np.array_equal(bp[7], c + r)
    assert np.array_equal(bp[1], c + np.float32([-r, -r, r])) and np.array_equal(bp[2], c + np.float32([r, -r, -r]))
    assert np.array_equal(bp[4], c + np.float32([-r, r, -r]))


def test_merge_and_add_voxels(config3):
    a, b = config3
    ka, ca = a.get_voxels()
    kb, cb = b.get_voxels()
    want = V.merge(ka, ca, kb, cb, True)
    s = a + b
    same(s, *want)
    assert len(want[0]) < len(ka) + len(kb)  # they overlap
    t = G.VoxelGrid()
    t.voxel_size, t.origin, t.voxels_keys, t.voxels_colors = a.voxel_size, a.origin, a.voxels_keys, a.voxels_colors
    t += b
    same(t, *want)
    u = a.select_by_index(np.arange(len(a)))
    u.add_voxels(kb, cb)
    same(u, *V.merge(ka, ca, kb, cb, False))
    # assigned keys that repeat, in any order: the stated left-to-right order defines the colours
    rng = np.random.default_rng(4)
    idx = rng.integers(0, len(ka), 300_000)
    r = a.select_by_index(idx)
    same(r + r, *V.merge(ka[idx], ca[idx], ka[idx], ca[idx], True))


def test_merge_rejects_mismatched_grids(config3):
    a, _ = config3
    c = G.VoxelGrid.create_dense((0.5, 0, 0), a.voxel_size, 0.1, 0.1, 0.1)
    with pytest.raises(ValueError):
        a + c
    d = G.VoxelGrid.create_dense(a.origin, 0.03, 0.1, 0.1, 0.1)
    with pytest.raises(ValueError):
        a + d
    wide = G.VoxelGrid()
    wide.voxel_size, wide.origin = a.voxel_size, a.origin
    wide.voxels_keys = np.array([[0, 0, 0], [3_000_000, 0, 0]], np.int32)  # a key span of 2^21 or more
    with pytest.raises(_lib.CphbError):
        wide.check_if_included(np.zeros((1, 3), np.float32))
    with pytest.raises(_lib.CphbError):
        wide + wide


def test_paint_select_invert(config3):
    a, _ = config3
    ka, ca = a.get_voxels()
    rng = np.random.default_rng(9)
    idx = rng.integers(0, len(ka), 500_000)
    g = a.select_by_index(np.arange(len(a)))
    g.paint_indexed_color(idx, (0.25, 0.5, 0.75))
    same(g, ka, V.paint(ca, idx, (0.25, 0.5, 0.75)))
    g.paint_uniform_color((0.1, 0.2, 0.3))
    same(g, ka, V.paint(ca, None, (0.1, 0.2, 0.3)))
    same(a.select_by_index(idx), *V.select(ka, ca, idx))
    same(a.select_by_index(idx, invert=True), *V.select(ka, ca, idx, True))
    same(a.select_by_index([], invert=True), ka, ca)
    assert len(a.select_by_index([])) == 0
    for bad in ([len(ka)], [-1], [0, 1, len(ka) + 5]):
        with pytest.raises(_lib.CphbError):
            a.select_by_index(bad)
        with pytest.raises(_lib.CphbError):
            a.select_by_index(bad, invert=True)
        with pytest.raises(_lib.CphbError):
            g.paint_indexed_color(bad, (1, 0, 0))
    same(g, ka, V.paint(ca, None, (0.1, 0.2, 0.3)))  # a refused paint changes nothing


def params(K, E, w, h):
    intr = CAM.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    return CAM.PinholeCameraParameters(intr, E)


@pytest.mark.parametrize("res,views", [(128, 8), (256, 16)])
@pytest.mark.parametrize("kind", ["depth", "mask"])
@pytest.mark.parametrize("keep", [False, True])
def test_carving_matches_oracle(res, views, kind, keep):
    w, h = 120, 96
    g = G.VoxelGrid.create_dense((-1, -1, -1), 2.0 / res, 2, 2, 2)
    keys, cols = g.get_voxels()
    for K, E in ring_cameras(views, w, h):
        depth = sphere_depth(K, E, w, h, 0.8)
        img = depth if kind == "depth" else (depth > 0).astype(np.uint8) * 255
        carve = g.carve_depth_map if kind == "depth" else g.carve_silhouette
        carve(G.Image(img), params(K, E, w, h), keep_voxels_outside_image=keep)
        keys, cols = V.carve(keys, cols, g.voxel_size, g.origin, img, K, E, keep)
        same(g, keys, cols)
    if kind == "mask":  # the reference's quirks: a uint8 mask removes everything, or keeps everything
        assert len(keys) == (res ** 3 if keep else 0)
    else:
        assert 0 < len(keys) < res ** 3


def test_carving_z_zero_and_nan_corners_are_outside():
    from test_oracle_voxelgrid_ops import nan_camera
    K, E = nan_camera()
    g = G.VoxelGrid.create_dense((0, 0, 0), 1.0, 1, 1, 2)
    cam = CAM.PinholeCameraParameters(CAM.PinholeCameraIntrinsic(8, 6, 0, 0, 3.5, 2.5), E)
    assert np.array_equal(cam.intrinsic.intrinsic_matrix, K)
    img = G.Image(np.full((6, 8), 100.0, np.float32))
    assert np.array_equal(g.carve_depth_map(img, cam, keep_voxels_outside_image=True).get_voxels()[0], [[0, 0, 0]])
    assert len(G.VoxelGrid.create_dense((0, 0, 0), 1.0, 1, 1, 2).carve_depth_map(img, cam)) == 0


def test_carving_rejects_mismatched_image():
    g = G.VoxelGrid.create_dense((-1, -1, -1), 0.25, 2, 2, 2)
    K, E = ring_cameras(1, 32, 32)[0]
    with pytest.raises(ValueError):
        g.carve_depth_map(G.Image(np.zeros((31, 32), np.float32)), params(K, E, 32, 32))
    with pytest.raises(ValueError):
        G.Image(np.zeros((4, 4), np.float64))


@pytest.fixture(scope="module")
def occ512():
    vs = 0.02
    scan = datagen.surface(1_000_000, 11, extent=4.0)[0] + np.array([0, 0, 0.5], np.float32)
    occ = G.OccupancyGrid(vs, 512, (2.0, 2.0, 0.5))
    occ.insert(G.PointCloud(scan.astype(np.float32)), (2.0, 2.0, 3.0))
    return occ


def test_create_from_occupancy_grid(occ512):
    occ = occ512
    cells, _ = occ.extract_occupied_voxels()
    assert len(cells) > 50_000
    vg = G.VoxelGrid.create_from_occupancy_grid(occ)
    same(vg, cells, np.tile(np.float32([0, 0, 1]), (len(cells), 1)))
    assert np.array_equal(vg.origin, V.occ_voxel_origin(512, occ.voxel_size, occ.origin))
    pc = G.PointCloud.create_from_occupancy_grid(occ)
    pts = V.occ_points(cells, 512, occ.voxel_size, occ.origin)
    assert np.array_equal(pc.points.cpu().view(np.uint32), pts.view(np.uint32))
    assert np.array_equal(pc.colors.cpu(), np.tile(np.float32([0, 0, 1]), (len(cells), 1)))
    # every voxel's centre is the point of the same cell (up to float32 rounding of the two expressions)
    centre = (cells.astype(np.float32) + np.float32(0.5)) * np.float32(vg.voxel_size) + vg.origin
    assert np.max(np.abs(centre - pts)) <= 4 * np.spacing(np.float32(8.0))
    # and every occupied cell of the map is reported against them (the query index of a cell is its linear index)
    res = cph.collision.compute_intersection(vg, occ)
    lin = (cells[:, 0].astype(np.int64) * 512 + cells[:, 1]) * 512 + cells[:, 2]
    assert np.array_equal(np.sort(res.get_second_collision_indices()), np.sort(lin))


def test_launch_counts_are_fixed_and_repeats_identical(config3, occ512):
    a, b = config3
    L = _lib.lib()
    small_a, small_b = a.select_by_index(np.arange(1000)), b.select_by_index(np.arange(500))
    K, E = ring_cameras(1, 64, 48)[0]
    img = G.Image(sphere_depth(K, E, 64, 48, 0.8))
    mask = G.Image(np.full((48, 64), 255, np.uint8))
    q = queries(10_000, 3)

    def calls(x, y):
        return {"dense": lambda: G.VoxelGrid.create_dense((0, 0, 0), 0.1, 1, 1, 1 if x is a else 0.5),
                "included": lambda: x.check_if_included(q),
                "merge": lambda: x + y,
                "add": lambda: x.select_by_index(np.arange(len(x))).add_voxels(y.get_voxels()[0]),
                "carve": lambda: x.select_by_index(np.arange(len(x))).carve_depth_map(img, params(K, E, 64, 48)),
                # no survivors: the same launches
                "carve_none": lambda: x.select_by_index(np.arange(len(x))).carve_silhouette(mask, params(K, E, 64, 48)),
                "select": lambda: x.select_by_index(np.arange(10)),
                "invert": lambda: x.select_by_index(np.arange(10), invert=True),
                "invert_all": lambda: x.select_by_index(np.arange(len(x)), invert=True),
                "paint": lambda: x.select_by_index(np.arange(len(x))).paint_indexed_color([1, 2], (0, 0, 0))}

    counts = {}
    for x, y in ((a, b), (small_a, small_b)):
        for name, fn in calls(x, y).items():
            fn()
            c0 = L.cphb_launch_count()
            r1 = fn()
            counts.setdefault(name, set()).add(L.cphb_launch_count() - c0)
            r2 = fn()
            if isinstance(r1, np.ndarray):
                assert np.array_equal(r1, r2)
            elif isinstance(r1, G.VoxelGrid):
                k1, c1 = r1.get_voxels()
                k2, c2 = r2.get_voxels()
                assert np.array_equal(k1, k2) and np.array_equal(c1.view(np.uint32), c2.view(np.uint32))
    assert all(len(v) == 1 for v in counts.values()), counts
    assert counts["carve_none"] == counts["carve"] and counts["invert_all"] == counts["invert"], counts
    v1 = G.VoxelGrid.create_from_occupancy_grid(occ512).get_voxels()
    v2 = G.VoxelGrid.create_from_occupancy_grid(occ512).get_voxels()
    assert np.array_equal(v1[0], v2[0]) and np.array_equal(v1[1], v2[1])
