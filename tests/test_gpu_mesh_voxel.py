"""GPU: VoxelGrid.create_from_triangle_mesh[_within_bounds] (csrc/voxelgrid.cu's triangle-major voxelisation) against
oracle/mesh_voxel.c bit for bit: random meshes, meshes extracted from TSDF sphere views and from the five real frames at
0.5x, 1x and 4x their voxel size, bounds that cut the mesh, a two-triangle 512^2 plane and a coarse 20-triangle solid in
a 512^3 grid, and the oracle's cell-major loop on the small inputs.  Also the output's form, the bounds of
create_from_triangle_mesh, repeats and the launch count, every rejection, and the grid feeding compute_edt and
compute_intersection."""
import ctypes
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import mesh_voxel_py as MV

G, CAM, I = cph.geometry, cph.camera, cph.integration
CT = I.TSDFVolumeColorType
VG = G.VoxelGrid
HERE = os.path.dirname(os.path.abspath(__file__))


def sphere_mesh(res=128, views=8):
    """test_gpu_mesh_ops.py's recipe: a radius-0.6 sphere seen from a ring of cameras, fused into a 2 m volume"""
    w, h = 160, 120
    vol = I.UniformTSDFVolume(2.0, res, 0.06, CT.RGB8)
    rng = np.random.default_rng(res)
    for K, E in ring_cameras(views, w, h, 2.5):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)), G.Image(d16),
                                                     1000.0, 100.0, False)
        vol.integrate(im, CAM.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    return vol.extract_triangle_mesh()


def real_mesh():
    """test_gpu_mesh_ops.py's recipe: the five real depth frames fused into an 8 m volume"""
    g = np.load(os.path.join(HERE, "golden", "tsdf_rgbd_known.npz"))
    K = CAM.PinholeCameraIntrinsic(CAM.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    vol = I.UniformTSDFVolume(8.0, 200, 0.04, CT.RGB8)
    rng = np.random.default_rng(5)
    for i in range(5):
        color = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(color), G.Image(g["depth"][i]), 1000.0, 4.0, False)
        vol.integrate(im, K, g["extrinsics"][i])
    return vol.extract_triangle_mesh()


def random_mesh(seed, nv=400, nt=600, scale=1.0):
    rng = np.random.default_rng(seed)
    v = (rng.normal(size=(nv, 3)) * scale).astype(np.float32)
    t = rng.integers(0, nv, (nt, 3)).astype(np.int32)
    t[3] = (t[3, 0], t[3, 0], t[3, 2])  # a segment
    t[4] = (t[4, 0], t[4, 0], t[4, 0])  # a point
    return v, t


def icosahedron(r, c):
    p = (1 + 5 ** 0.5) / 2
    v = np.array([[-1, p, 0], [1, p, 0], [-1, -p, 0], [1, -p, 0], [0, -1, p], [0, 1, p], [0, -1, -p], [0, 1, -p], [p, 0, -1],
                  [p, 0, 1], [-p, 0, -1], [-p, 0, 1]], np.float64)
    v = v / np.linalg.norm(v[0]) * r + c
    t = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
         [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    return v.astype(np.float32), np.array(t, np.int32)


@pytest.fixture(scope="module")
def meshes():
    out = {}
    for name, m in (("sphere", sphere_mesh()), ("real", real_mesh())):
        out[name] = (m.vertices.cpu(), m.triangles.cpu())
    return out


def device(v, t, vs, mn, mx):
    g = VG.create_from_triangle_mesh_within_bounds(G.TriangleMesh(v, t), vs, mn, mx)
    keys, cols = g.get_voxels()
    return g, keys, cols


def check_against_oracle(v, t, vs, mn, mx, cell_major=False):
    g, keys, cols = device(v, t, vs, mn, mx)
    want = MV.voxelize(v, t, vs, mn, mx, MV.TRIANGLE_MAJOR)
    assert keys.dtype == np.int32 and np.array_equal(keys, want), (len(keys), len(want))
    if cell_major:
        assert np.array_equal(MV.voxelize(v, t, vs, mn, mx, MV.CELL_MAJOR), want)
    assert np.array_equal(cols, np.ones((len(keys), 3), np.float32))
    assert g.voxel_size == float(np.float32(vs)) and np.array_equal(g.origin, np.asarray(mn, np.float32))
    if len(keys) > 1:  # unique, lexicographic
        d = np.diff(keys.astype(np.int64) @ np.array([1 << 42, 1 << 21, 1], np.int64))
        assert (d > 0).all()
    return keys


@pytest.mark.parametrize("seed", range(4))
def test_random_meshes_match_the_oracle(seed):
    v, t = random_mesh(seed)
    keys = check_against_oracle(v, t, 0.11, (-3, -3, -3), (3, 3, 3))
    assert len(keys) > 1000


@pytest.mark.parametrize("seed", range(3))
def test_small_random_meshes_match_the_cell_major_loop(seed):
    v, t = random_mesh(100 + seed, 30, 25, 0.6)
    v[0] = (np.nan, 0, 0)
    v[1] = (np.inf, 0, 0)
    check_against_oracle(v, t, 0.125, (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5), cell_major=True)


def test_dyadic_lattice_vertices_on_faces_edges_and_corners():
    rng = np.random.default_rng(7)
    v = (rng.integers(-16, 17, (60, 3)) / 8.0).astype(np.float32)
    t = rng.integers(0, 60, (80, 3)).astype(np.int32)
    check_against_oracle(v, t, 0.125, (-2, -2, -2), (2, 2, 2), cell_major=True)


@pytest.mark.parametrize("name", ["sphere", "real"])
@pytest.mark.parametrize("factor", [0.5, 1.0, 4.0])
def test_tsdf_meshes_match_the_oracle(meshes, name, factor):
    v, t = meshes[name]
    vs = (2.0 / 128 if name == "sphere" else 8.0 / 200) * factor
    m = G.TriangleMesh(v, t)
    mn, mx = m.get_min_bound(), m.get_max_bound()
    h = np.float32(vs) * np.float32(0.5)
    keys = check_against_oracle(v, t, vs, mn - h, mx + h)
    assert len(keys) > 100


def test_bounds_that_cut_the_mesh(meshes):
    v, t = meshes["sphere"]
    check_against_oracle(v, t, 0.02, (-0.31, -0.7, 0.05), (0.4, 0.17, 0.73))
    check_against_oracle(v, t, 0.02, (0.61, 0.61, 0.61), (1.0, 1.0, 1.0))  # misses the mesh


def test_load_balance_cases_at_512():
    # a two-triangle plane across a 512^2 grid, tilted so each column meets 2 or 3 cells
    v = np.array([[0.1, 0.1, 3.2], [511.9, 0.1, 4.9], [0.1, 511.9, 3.7], [511.9, 511.9, 5.3]], np.float32)
    t = np.array([[0, 1, 2], [1, 3, 2]], np.int32)
    keys = check_against_oracle(v, t, 1.0, (0, 0, 0), (512, 512, 10))
    assert len(keys) >= 512 * 512
    # a coarse 20-triangle solid filling most of a 512^3 grid
    v, t = icosahedron(200.0, np.array([256.3, 255.7, 256.1]))
    keys = check_against_oracle(v, t, 1.0, (0, 0, 0), (512, 512, 512))
    assert len(keys) > 100000


def test_create_from_triangle_mesh_uses_the_vertex_bounds(meshes):
    v, t = meshes["sphere"]
    m = G.TriangleMesh(v, t)
    assert np.array_equal(m.get_min_bound(), v.min(0)) and np.array_equal(m.get_max_bound(), v.max(0))
    vs = np.float32(0.03)
    g = VG.create_from_triangle_mesh(m, vs)
    lo = v.min(0) - vs * np.float32(0.5)
    assert np.array_equal(g.origin, lo)
    assert np.array_equal(g.get_voxels()[0], MV.voxelize(v, t, vs, lo, v.max(0) + vs * np.float32(0.5)))
    e = VG.create_from_triangle_mesh(G.TriangleMesh(), 0.5)
    assert len(e) == 0 and e.voxel_size == 0.5 and np.array_equal(e.origin, np.full(3, -0.25, np.float32))
    e = VG.create_from_triangle_mesh_within_bounds(G.TriangleMesh(v, np.zeros((0, 3), np.int32)), 0.1, (0, 1, 2), (1, 2, 3))
    assert len(e) == 0 and np.array_equal(e.origin, np.float32([0, 1, 2]))


def test_the_cell_centre_rule():
    """deviation 1: a triangle in the plane z = o_z + 0.75 vs is in cell k_z = 0, the cell get_voxel gives"""
    v = np.array([[0.1, 0.1, 0.375], [1.9, 0.1, 0.375], [0.1, 1.9, 0.375]], np.float32)
    g, keys, _ = device(v, np.array([[0, 1, 2]], np.int32), 0.5, (0, 0, 0), (2, 2, 2))
    assert set(keys[:, 2]) == {0}
    assert np.array_equal(g.get_voxel(v[0]), [0, 0, 0])
    assert set(MV.voxelize(v, [[0, 1, 2]], 0.5, (0, 0, 0), (2, 2, 2), MV.CELL_MAJOR, corner=True)[:, 2]) == {1}


def test_repeats_are_bit_identical_and_the_launch_count_fixed(meshes):
    v, t = meshes["real"]
    m = G.TriangleMesh(v, t)
    L = _lib.lib()
    counts, outs = [], []
    lo = m.get_min_bound()
    for off in (0.0, 0.0, 100.0):  # the last grid misses the mesh: its sizing call finds 0 voxels and stops there
        n0 = L.cphb_launch_count()
        outs.append(VG.create_from_triangle_mesh_within_bounds(m, 8.0 / 256, lo + off, lo + off + 8.0).get_voxels()[0])
        counts.append(L.cphb_launch_count() - n0)
    assert np.array_equal(outs[0], outs[1]) and len(outs[0]) > 0 and len(outs[2]) == 0
    # per call: setup, CUB's 2 scan kernels, count, block scan, write, the 24-bit key sort (3 passes + histogram),
    # unique count, block scan, unique write; the Python path sizes, then writes
    per_call = 1 + 2 + 3 + (3 + 1) + 3
    assert counts == [2 * per_call, 2 * per_call, per_call], counts


def _pool_used():
    """the bytes in use in the device's default memory pool, which the library allocates from, once the stream's
    pending frees have run"""
    _lib.check(_lib.lib().cphb_stream_synchronize(None))
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool, used = ctypes.c_int(), ctypes.c_void_p(), ctypes.c_uint64()
    assert cu.cuCtxGetDevice(ctypes.byref(dev)) == 0
    assert cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, 7, ctypes.byref(used)) == 0  # CU_MEMPOOL_ATTR_USED_MEM_CURRENT
    return used.value


def test_every_rejection_raises_and_leaves_nothing_allocated():
    v, t = random_mesh(3, 50, 40)
    m = G.TriangleMesh(v, t)
    VG.create_from_triangle_mesh_within_bounds(m, 0.1, (-1, -1, -1), (1, 1, 1))
    bad_index = t.copy()
    bad_index[17, 1] = 50
    neg = t.copy()
    neg[39, 2] = -1
    cases = [(G.TriangleMesh(v, bad_index), 0.1, (-1, -1, -1), (1, 1, 1)), (G.TriangleMesh(v, neg), 0.1, (-1, -1, -1), (1, 1, 1)),
             (m, 0.0, (-1, -1, -1), (1, 1, 1)), (m, -0.1, (-1, -1, -1), (1, 1, 1)), (m, float("nan"), (-1, -1, -1), (1, 1, 1)),
             (m, float("inf"), (-1, -1, -1), (1, 1, 1)), (m, 0.1, (-1, float("nan"), -1), (1, 1, 1)),
             (m, 0.1, (-1, -1, -1), (1, float("inf"), 1)), (m, 0.1, (1, 1, 1), (-1, 1, 1)),
             (m, 1.0, (0, 0, 0), (2.0 ** 21, 1, 1)), (m, 1.0, (0, 0, 0), (1, 1, 2.0 ** 21 - 0.5))]
    used = _pool_used()  # the meshes above are allocated: from here on every call must give back what it takes
    for mesh, vs, lo, hi in cases:
        with pytest.raises(_lib.CphbError):
            VG.create_from_triangle_mesh_within_bounds(mesh, vs, lo, hi)
        assert _pool_used() == used
    g = VG.create_from_triangle_mesh_within_bounds(m, 1.0, (0, 0, 0), (1, 1, 2.0 ** 21 - 1.5))  # the largest count passes
    assert g.voxel_size == 1.0


def test_downstream_distance_transform_and_collision(meshes):
    v, t = meshes["sphere"]
    m = G.TriangleMesh(v, t)
    size, res = 2.0, 128
    vs = size / res
    grid = VG.create_from_triangle_mesh_within_bounds(m, vs, (-1, -1, -1), (1, 1, 1))
    dt = G.DistanceTransform(vs, res)
    dt.compute_edt(grid)
    assert abs(dt.get_distance((0.0, 0.0, 0.0)) - 0.6) < 2 * vs
    samples = m.sample_points_uniformly(50000)
    pts = VG.create_from_point_cloud_within_bounds(samples, vs, (-1, -1, -1), (1, 1, 1))
    hit = cph.collision.compute_intersection(grid, pts, 0.0)  # each query voxel reports the first target voxel it hits
    assert len(np.unique(hit.get_second_collision_indices())) == len(pts)
