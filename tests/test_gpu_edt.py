"""GPU: geometry::DistanceTransform (csrc/edt.cu).

- The device equals the CPU oracle (oracle/edt.c) bit for bit on every cell -- nearest index, state and distance bits --
  at resolutions 1, 7, 100, 257 and 512, for VoxelGrids of datagen surfaces and for random sparse and dense sets and
  lattices, through both ComputeEDT and ComputeVoronoiDiagram.  At 1024^3, sampled cells against a brute force.
- create_from_occupancy_grid after insert, add_voxels and set_free_area; get_distance, get_distances and get_voxel
  including queries outside the grid and NaN; reconstruct; a repeated compute equals a fresh one; to_torch is zero-copy.
- A compute is a fixed number of launches whatever the resolution and the site count; illegal arguments are refused."""
import ctypes as C

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing import datagen
from cupoch_b200.utility import DeviceArray
from test_oracle_edt import grid_cells

G = cph.geometry


@pytest.fixture(scope="module")
def E():
    from oracle import edt_py
    edt_py.build()
    return edt_py


def device_grid(dt):
    """-> (nearest [r, r, r, 3] uint16, state [r, r, r] uint8, distance [r, r, r] float32) of the device grid"""
    r = dt.resolution
    L = _lib.lib()
    p = DeviceArray((r, r, r), np.uint32, ptr=L.cphb_dt_nearest_data(dt._h), base=dt).cpu()
    d = DeviceArray((r, r, r), np.float32, ptr=L.cphb_dt_distance_data(dt._h), base=dt).cpu()
    near = np.stack([(p >> 20) & 1023, (p >> 10) & 1023, p & 1023], -1).astype(np.uint16)
    state = np.where(p & (1 << 30), 2, 0).astype(np.uint8)
    assert not (p >> 31).any()
    return near, state, d


def assert_same(dev, orc):
    for name, a, b in zip(("nearest", "state", "distance"), dev, orc):
        if b.dtype == np.float32:
            a, b = a.view(np.uint32), b.view(np.uint32)
        bad = np.flatnonzero((a != b).reshape(a.shape[0] ** 3, -1).any(1))
        assert bad.size == 0, "%s differs at %d cells, first %s: %s vs %s" % (
            name, bad.size, np.unravel_index(bad[0], a.shape[:3]), a.reshape(-1, *a.shape[3:])[bad[0]], b.reshape(-1, *b.shape[3:])[bad[0]])


def site_sets(r, seed):
    rng = np.random.default_rng(seed)
    step = max(1, r // 5)
    g = np.arange(1, r, step)
    sets = {"sparse": rng.integers(0, r, (max(1, r ** 3 // 5000), 3)),
            "lattice": np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)}
    if r <= 257:
        sets["dense"] = rng.integers(-2, r + 2, (r ** 3 // 3 + 1, 3))  # with some outside the grid
    return sets


@pytest.mark.parametrize("r", [1, 7, 100, 257, 512])
def test_sites_equal_oracle(E, r):
    vs = 0.03
    dt = G.DistanceTransform(vs, r)
    for name, sites in site_sets(r, r).items():
        for with_distance in (True, False):
            (dt.compute_edt if with_distance else dt.compute_voronoi_diagram)(sites.astype(np.int32))
            assert_same(device_grid(dt), E.compute(r, sites, vs, with_distance))


@pytest.mark.parametrize("r,vg_vs,extent", [(7, 0.2, 1.0), (100, 0.01, 1.0), (257, 0.004, 1.0), (512, 0.004, 2.0)])
def test_voxel_grid_equals_oracle(E, r, vg_vs, extent):
    pts = datagen.surface(400_000, 31 + r, extent=extent)[0]
    vg = G.VoxelGrid.create_from_point_cloud(G.PointCloud(pts), vg_vs)
    assert len(vg) > 0
    origin = (0.5 * extent, 0.5 * extent, 0.01)
    dt = G.DistanceTransform(vg_vs, r, origin)
    keys = vg.voxels_keys.cpu()
    for with_distance in (True, False):
        (dt.compute_edt if with_distance else dt.compute_voronoi_diagram)(vg)
        assert_same(device_grid(dt), E.compute_voxel_grid(r, vg_vs, origin, keys, vg.voxel_size, vg.origin, with_distance))


def test_voxel_size_mismatch_is_logged_and_changes_nothing(E, capfd):
    dt = G.DistanceTransform(0.05, 16)
    dt.compute_edt(np.array([[3, 4, 5]], np.int32))
    before = device_grid(dt)
    vg = G.VoxelGrid.create_from_point_cloud(G.PointCloud(datagen.surface(1000, 3)[0]), 0.1)
    dt.compute_edt(vg)
    assert "different voxel size" in capfd.readouterr().err
    for a, b in zip(device_grid(dt), before):
        np.testing.assert_array_equal(a, b)


def test_1024_sampled_cells_against_brute_force():
    r = 1024
    rng = np.random.default_rng(9)
    sites = np.unique(rng.integers(0, r, (300, 3)), axis=0)  # lexicographic order: argmin takes the smallest
    dt = G.DistanceTransform(1.0, r)
    dt.compute_edt(sites.astype(np.int32))
    L = _lib.lib()
    cells = np.concatenate([rng.integers(0, r, (20000, 3)), [[0, 0, 0], [r - 1, r - 1, r - 1], [0, r - 1, 0]]])
    lin = (cells[:, 0] * r + cells[:, 1]) * r + cells[:, 2]
    # gather the sampled cells on the device through torch (the whole grid is 8 GB)
    import torch
    p = torch.as_tensor(DeviceArray((r ** 3,), np.int32, ptr=L.cphb_dt_nearest_data(dt._h), base=dt), device="cuda")
    got = p[torch.as_tensor(lin, device="cuda")].cpu().numpy().astype(np.int64)
    d = dt.to_torch().reshape(-1)[torch.as_tensor(lin, device="cuda")].cpu().numpy()
    D = ((cells[:, None, :].astype(np.int64) - sites[None]) ** 2).sum(-1)
    a = np.argmin(D, 1)
    want = sites[a]
    np.testing.assert_array_equal(np.stack([(got >> 20) & 1023, (got >> 10) & 1023, got & 1023], -1), want)
    assert not (got & (1 << 30)).any()
    np.testing.assert_array_equal(d, np.sqrt(D[np.arange(len(a)), a].astype(np.float32)))


def test_no_sites_and_outside_sites(E):
    r, vs = 33, 0.1
    dt = G.DistanceTransform(vs, r)
    dt.compute_edt(np.array([[-1, 0, 0], [r, 1, 1], [0, 0, 40]], np.int32))
    assert_same(device_grid(dt), E.compute(r, np.zeros((0, 3)), vs))
    dt.compute_voronoi_diagram(np.zeros((0, 3), np.int32))
    assert_same(device_grid(dt), E.compute(r, np.zeros((0, 3)), vs, with_distance=False))


def test_fresh_grid_and_reconstruct(E):
    dt = G.DistanceTransform(0.5, 9)
    assert_same(device_grid(dt), E.default_grid(9))
    dt.compute_edt(np.array([[1, 2, 3], [8, 0, 8]], np.int32))
    g = E.compute(9, [[1, 2, 3], [8, 0, 8]], 0.5)
    for r_new in (5, 12):
        dt.reconstruct(0.25, r_new)
        assert dt.resolution == r_new and dt.voxel_size == 0.25
        g = E.reconstruct(g, r_new)
        assert_same(device_grid(dt), g)
    dt.compute_edt(np.array([[0, 0, 0]], np.int32))  # the new voxel size applies from here on
    assert_same(device_grid(dt), E.compute(12, [[0, 0, 0]], 0.25))


def test_repeated_compute_equals_fresh(E):
    r = 64
    rng = np.random.default_rng(3)
    a, b = rng.integers(0, r, (4000, 3)).astype(np.int32), rng.integers(0, r, (7, 3)).astype(np.int32)
    dt = G.DistanceTransform(0.1, r)
    dt.compute_edt(a)
    dt.compute_edt(b)
    fresh = G.DistanceTransform(0.1, r)
    fresh.compute_edt(b)
    for x, y in zip(device_grid(dt), device_grid(fresh)):
        np.testing.assert_array_equal(x, y)
    assert_same(device_grid(dt), E.compute(r, b, 0.1))


def test_occupancy_grid(E):
    r, vs = 64, 0.05
    occ = G.OccupancyGrid(vs, r, (0.1, 0.0, 0.0))
    pts = datagen.surface(20000, 5)[0] - np.float32(0.5)
    occ.insert(G.PointCloud(pts), (0.0, 0.0, 1.0))
    occ.add_voxels(np.array([[1, 2, 3], [60, 60, 60], [60, 60, 60]], np.int32), occupied=True)
    occ.set_free_area((-1.6, -1.6, -1.6), (-1.0, -1.0, -1.0))
    occ.occ_prob_thres_log = 0.5
    dt = G.DistanceTransform.create_from_occupancy_grid(occ)
    assert dt.resolution == r and dt.voxel_size == np.float32(vs) and np.array_equal(dt.origin, occ.origin)
    prob = occ.to_torch().cpu().numpy()
    sites = E.occupied_cells(prob, 0.5)
    assert 10 < len(sites) < r ** 3 // 10
    assert_same(device_grid(dt), E.compute(r, sites, vs))
    p = _lib.OccGridParams()
    _lib.check(_lib.lib().cphb_occgrid_get_params(occ._h, C.byref(p)))
    assert p.occ_prob_thres_log == np.float32(0.5) and p.prob_hit_log == np.float32(0.85)


def test_queries(E):
    r, vs, origin = 40, 0.25, np.array([0.5, -1.0, 2.0], np.float32)
    rng = np.random.default_rng(11)
    sites = rng.integers(0, r, (100, 3)).astype(np.int32)
    dt = G.DistanceTransform(vs, r, origin)
    dt.compute_edt(sites)
    nearest, state, dist = E.compute(r, sites, vs)
    q = (rng.uniform(-6, 6, (100_000, 3)) + origin).astype(np.float32)
    q[:4] = [[np.nan, 0, 0], [0, np.inf, 0], [100, 0, 0], origin]
    d = dt.get_distances(q)
    assert isinstance(d, DeviceArray) and d.dtype == np.float32
    want = E.get_distances(dist, q, vs, origin)
    np.testing.assert_array_equal(d.cpu().view(np.uint32), want.view(np.uint32))
    import torch
    np.testing.assert_array_equal(dt.get_distances(torch.as_tensor(q, device="cuda")).cpu(), d.cpu())
    assert d.cpu()[:3].tolist() == [0.0, 0.0, 0.0]
    for i in list(range(8)) + list(rng.integers(0, len(q), 200)):
        assert dt.get_distance(q[i]) == want[i]
        found, v = dt.get_voxel(q[i])
        k = E.voxel_index(q[i:i + 1], vs, origin, r)[0]
        assert found == (k >= 0)
        if k >= 0:
            assert v.nearest_index.tolist() == nearest.reshape(-1, 3)[k].tolist()
            assert np.float32(v.distance).view(np.uint32) == dist.reshape(-1)[k].view(np.uint32)
        else:
            assert v.nearest_index.tolist() == [0, 0, 0] and v.distance == 0.0
    # origin and voxel size are read at every query
    dt.origin = origin + np.float32(1.0)
    np.testing.assert_array_equal(dt.get_distances(q).cpu(), E.get_distances(dist, q, vs, origin + np.float32(1.0)))


def test_to_torch_zero_copy_and_repeatable():
    import torch
    r = 100
    sites = np.random.default_rng(2).integers(0, r, (5000, 3)).astype(np.int32)
    dt = G.DistanceTransform(0.02, r)
    dt.compute_edt(sites)
    t = dt.to_torch()
    assert t.shape == (r, r, r) and t.dtype == torch.float32 and t.is_cuda
    assert t.data_ptr() == _lib.lib().cphb_dt_distance_data(dt._h)
    first = t.clone()
    for _ in range(3):
        dt.compute_edt(sites)
        assert torch.equal(dt.to_torch(), first)
        assert torch.equal(t, first)


def test_launch_count_is_fixed():
    L = _lib.lib()
    rng = np.random.default_rng(4)
    deltas = set()
    for r in (64, 512):
        dt = G.DistanceTransform(1.0, r)
        for n in (1, 1_000_000):
            d = DeviceArray.from_numpy(rng.integers(0, r, (n, 3)), np.int32)
            for with_distance in (1, 0):
                c0 = L.cphb_launch_count()
                _lib.check(L.cphb_dt_compute_sites(dt._h, d.ptr, n, with_distance, None))
                deltas.add(L.cphb_launch_count() - c0)
        _lib.check(L.cphb_stream_synchronize(None))
    assert deltas == {4}  # stamp + three sweeps (the clear is a memset)


def test_illegal_arguments():
    L = _lib.lib()
    for r in (0, 1025, -3):
        with pytest.raises(_lib.CphbError):
            G.DistanceTransform(0.05, r)
    dt = G.DistanceTransform(0.05, 8)
    with pytest.raises(_lib.CphbError):
        dt.reconstruct(0.05, 1025)
    assert dt.resolution == 8
    h = C.c_void_p()
    assert L.cphb_dt_create(0.05, 0, None, None, C.byref(h)) == _lib.CPHB_ERR_INVALID
    assert L.cphb_dt_compute_sites(None, None, 0, 1, None) == _lib.CPHB_ERR_INVALID
    assert L.cphb_dt_compute_voxel_grid(None, None, 0, 0.05, (C.c_float * 3)(), 1, None) == _lib.CPHB_ERR_INVALID
    assert L.cphb_dt_get_distances(None, None, 0, None, None) == _lib.CPHB_ERR_INVALID
    assert L.cphb_dt_reconstruct(None, 0.05, 8, None) == _lib.CPHB_ERR_INVALID
    assert L.cphb_dt_from_occgrid(None, None, C.byref(h)) == _lib.CPHB_ERR_INVALID
    f = C.c_int(0)
    assert L.cphb_dt_get_voxel(None, (C.c_float * 3)(), C.byref(f), None, None, None, None) == _lib.CPHB_ERR_INVALID
    assert L.cphb_dt_distance_data(None) is None and L.cphb_dt_nearest_data(None) is None
    big = G.OccupancyGrid(0.05, 1030)
    with pytest.raises(_lib.CphbError):
        G.DistanceTransform.create_from_occupancy_grid(big)
