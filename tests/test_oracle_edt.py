"""CPU: the DistanceTransform restatement (oracle/edt.c) that tests/test_gpu_edt.py holds the device to.

- On every cell it equals a numpy brute force: the argmin of the integer d2 over all sites, the lexicographically smallest
  (x, y, z) among equal ones, at resolutions 1, 2, 7, 9, 24 and 33, for random, dense, single-site and all-sites sets and
  tie-heavy lattices.
- On a 128^3 grid its d2 equals round(scipy.ndimage.distance_transform_edt(...)^2), an independent implementation.
- The reference's own unit test (src/tests/geometry/distancetransform.cpp:32-46).
- One test per mirrored quirk and per deviation of DESIGN.md parity hazard 13."""
import numpy as np
import pytest

from oracle import edt_py as E

BRUTE_CHUNK = 1 << 22  # cells x sites per numpy block


def grid_cells(r):
    g = np.arange(r)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


def brute(r, sites):
    """-> (nearest [r, r, r, 3], d2 [r, r, r]) with the lexicographic tie rule (argmin over lexsorted unique sites)"""
    s = np.unique(np.asarray(sites, np.int64).reshape(-1, 3), axis=0)
    g = grid_cells(r).astype(np.int64)
    near = np.empty_like(g)
    d2 = np.empty(len(g), np.int64)
    step = max(1, BRUTE_CHUNK // len(s))
    for lo in range(0, len(g), step):
        D = ((g[lo:lo + step, None, :] - s[None, :, :]) ** 2).sum(-1)
        a = np.argmin(D, 1)  # the first minimum: the lexicographically smallest site
        near[lo:lo + step] = s[a]
        d2[lo:lo + step] = D[np.arange(len(a)), a]
    return near.reshape(r, r, r, 3), d2.reshape(r, r, r)


def site_sets(r, seed):
    rng = np.random.default_rng(seed)
    sets = {"single": rng.integers(0, r, (1, 3)),
            "random": rng.integers(0, r, (max(1, r ** 3 // 200) + 3, 3))}
    step = max(1, r // 4)
    g = np.arange(0, r, step)
    sets["lattice"] = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)  # equidistant sites everywhere
    sets["planes"] = np.concatenate([grid_cells(r)[grid_cells(r)[:, 0] == 0], grid_cells(r)[grid_cells(r)[:, 1] == r - 1]])
    if r <= 24:
        sets["dense"] = rng.integers(0, r, (r ** 3 // 2 + 1, 3))
    return sets


@pytest.mark.parametrize("r", [1, 2, 7, 9, 24, 33])
def test_oracle_equals_brute_force(r):
    for name, sites in site_sets(r, 100 + r).items():
        nearest, state, dist = E.compute(r, sites, voxel_size=1.0)
        b_near, b_d2 = brute(r, sites)
        np.testing.assert_array_equal(nearest.astype(np.int64), b_near, err_msg="%d %s" % (r, name))
        assert (state == 0).all()
        np.testing.assert_array_equal(dist, np.sqrt(b_d2.astype(np.float32)), err_msg="%d %s" % (r, name))
        vn, vs, vd = E.compute(r, sites, voxel_size=1.0, with_distance=False)  # ComputeVoronoiDiagram
        np.testing.assert_array_equal(vn, nearest)
        assert (vd == 0).all() and (vs == 0).all()


@pytest.mark.parametrize("r", [1, 7, 33])
def test_all_sites_is_identity(r):
    nearest, state, dist = E.compute(r, grid_cells(r), voxel_size=0.5)
    np.testing.assert_array_equal(nearest.reshape(-1, 3), grid_cells(r))
    assert (dist == 0).all() and (state == 0).all()


def test_tie_takes_lexicographically_smallest():
    # cell (2, 2, 2) is at d2 = 4 from all six axis neighbours two cells away; (0, 2, 2) is the smallest
    six = np.array([[0, 2, 2], [4, 2, 2], [2, 0, 2], [2, 4, 2], [2, 2, 0], [2, 2, 4]])
    for order in (six, six[::-1], six[[3, 1, 5, 0, 4, 2]]):
        nearest, _, dist = E.compute(5, order)
        assert nearest[2, 2, 2].tolist() == [0, 2, 2] and dist[2, 2, 2] == 2.0


def test_d2_equals_scipy_edt_128():
    from scipy import ndimage
    r = 128
    rng = np.random.default_rng(7)
    sites = rng.integers(0, r, (3000, 3))
    mask = np.ones((r, r, r), bool)
    mask[tuple(sites.T)] = False
    ref = np.rint(ndimage.distance_transform_edt(mask) ** 2).astype(np.int64)
    nearest, _, dist = E.compute(r, sites, voxel_size=1.0)
    d2 = ((nearest.astype(np.int64) - grid_cells(r).reshape(r, r, r, 3)) ** 2).sum(-1)
    np.testing.assert_array_equal(d2, ref)
    np.testing.assert_array_equal(dist, np.sqrt(ref.astype(np.float32)))


def test_reference_unit_test():
    # distancetransform.cpp:32-46: VoxelGrid voxel 1.0 with key (5,5,5), DistanceTransform(1.0, 512), ComputeVoronoiDiagram,
    # GetVoxel((0,0,0)) is found and its nearest index is (5,5,5) + 512 / 2
    r = 512
    cells, inside = E.key_cells(np.array([[5, 5, 5]]), 1.0, (0, 0, 0), (0, 0, 0), r)
    assert inside.all() and cells.tolist() == [[261, 261, 261]]
    nearest, state, dist = E.compute_voxel_grid(r, 1.0, (0, 0, 0), [[5, 5, 5]], 1.0, (0, 0, 0), with_distance=False)
    i = E.voxel_index([[0.0, 0.0, 0.0]], 1.0, (0, 0, 0), r)[0]
    assert i == (256 * r + 256) * r + 256
    assert nearest.reshape(-1, 3)[i].tolist() == [261, 261, 261] and state.reshape(-1)[i] == 0 and dist.reshape(-1)[i] == 0


def test_voxel_size_mismatch_leaves_grid_unchanged():
    eps = np.finfo(np.float32).eps
    assert E.voxel_size_ok(0.5, 0.5) and E.voxel_size_ok(1.0, 1.0 + eps)
    assert not E.voxel_size_ok(1.0, 1.0 + 2 * eps) and not E.voxel_size_ok(0.05, 0.1)
    assert E.compute_voxel_grid(8, 0.05, (0, 0, 0), [[0, 0, 0]], 0.1, (0, 0, 0)) is None


def test_no_sites():
    # with no site, every nearest is (0,0,0) with NotSite and the distance is |cell| * voxel_size (0 for Voronoi only)
    r, vs = 6, 0.25
    nearest, state, dist = E.compute(r, np.zeros((0, 3)), voxel_size=vs)
    assert (nearest == 0).all() and (state == E.NOT_SITE).all()
    c = grid_cells(r).reshape(r, r, r, 3)
    np.testing.assert_array_equal(dist, np.sqrt((c ** 2).sum(-1).astype(np.float32)) * np.float32(vs))
    _, _, vd = E.compute(r, np.zeros((0, 3)), voxel_size=vs, with_distance=False)
    assert (vd == 0).all()
    # sites that are all outside the grid are no sites
    n2, s2, d2 = E.compute(r, [[-1, 0, 0], [0, r, 0], [0, 0, 99]], voxel_size=vs)
    assert (s2 == E.NOT_SITE).all() and np.array_equal(d2, dist)


def test_sites_outside_grid_are_ignored():
    r = 9
    inside = np.array([[1, 2, 3], [7, 7, 0]])
    outside = np.array([[-1, 2, 3], [9, 0, 0], [0, -5, 4], [2, 2, 9], [1 << 20, 0, 0]])
    a = E.compute(r, np.concatenate([inside, outside]))
    b = E.compute(r, inside)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_reconstruct_keeps_linear_prefix():
    g = E.compute(4, [[1, 1, 1]], voxel_size=0.5)
    small = E.reconstruct(g, 3)  # the first 27 cells of the 4^3 grid, in linear order
    np.testing.assert_array_equal(small[0].reshape(-1, 3), g[0].reshape(-1, 3)[:27])
    np.testing.assert_array_equal(small[2].reshape(-1), g[2].reshape(-1)[:27])  # distances are not rescaled
    big = E.reconstruct(g, 5)
    np.testing.assert_array_equal(big[0].reshape(-1, 3)[:64], g[0].reshape(-1, 3))
    assert (big[0].reshape(-1, 3)[64:] == 0).all() and (big[1].reshape(-1)[64:] == E.NOT_SITE).all()
    assert (big[1].reshape(-1)[:64] == 0).all() and (big[2].reshape(-1)[64:] == 0).all()


def test_key_mapping_at_a_cell_face():
    # key * vs + o_vg - o_dt lands exactly on a cell face: floor keeps it in the upper cell; just below goes down
    r = 8
    cells, inside = E.key_cells([[2, -4, 0]], 0.5, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), r)
    assert cells.tolist() == [[6, 0, 4]] and inside.all()
    below = np.nextafter(np.float32(0), np.float32(-1))
    cells, inside = E.key_cells([[0, 0, 0]], 0.5, (below, 0.0, 0.0), (0.0, 0.0, 0.0), r)
    assert cells.tolist() == [[3, 4, 4]]
    cells, inside = E.key_cells([[4, -5, 0], [0, 0, 0]], 0.5, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), r)
    assert inside.tolist() == [False, True]  # 4 + 4 = 8 and -5 + 4 = -1 are outside


def test_query_mappings():
    r, vs, o = 8, 0.5, np.array([1.0, -2.0, 0.5], np.float32)
    # get_distance: floor(((q - o) + (0.5 * vs) * r) / vs); get_voxel: floor((q - o) / vs) + r / 2
    q = np.array([o, o + 0.26, o - 2.0, o + 1.99, o + 2.0, [np.nan, 0, 0], o - 2.01], np.float32)
    di = E.distance_index(q, vs, o, r)
    vi = E.voxel_index(q, vs, o, r)
    lin = lambda x, y, z: (x * r + y) * r + z
    assert di.tolist() == vi.tolist() == [lin(4, 4, 4), lin(4, 4, 4), 0, lin(7, 7, 7), -1, -1, -1]
    # the two formulas part where ((q - o) + 2) / vs and (q - o) / vs + 4 round differently
    q = np.array([[np.nextafter(o[0], np.float32(-np.inf)), o[1], o[2]]], np.float32)
    assert E.voxel_index(q, vs, o, r)[0] == lin(3, 4, 4) and E.distance_index(q, vs, o, r)[0] == lin(4, 4, 4)
    d = E.compute(r, [[0, 0, 0]], vs)[2]
    np.testing.assert_array_equal(E.get_distances(d, q, vs, o), d.reshape(-1)[[lin(4, 4, 4)]])
    assert E.get_distances(d, [[np.nan, 0, 0], [100, 0, 0]], vs, o).tolist() == [0.0, 0.0]
