"""GPU: UniformTSDFVolume.extract_triangle_mesh and TriangleMesh's normals (csrc/tsdf.cu, csrc/mesh.cu) against
oracle/tsdf_mesh.c bit for bit: the reference's five real frames, synthetic sphere views at all three colour types,
all 256 single-cube configurations and random fields written straight into the planes.  Also repeats, the launch
count, empty volumes, the sizing call and the index checks of the normal computations."""
import ctypes
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from cupoch_b200.utility import DeviceArray
from oracle import tsdf_mesh_py as M, tsdf_py as T

G, CAM, I = cph.geometry, cph.camera, cph.integration
CT = I.TSDFVolumeColorType
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsdf_rgbd_known.npz")


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def arrays(mesh):
    z3, zi = np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)
    v = mesh.vertices.cpu() if mesh.has_vertices() else z3
    t = mesh.triangles.cpu() if mesh.has_triangles() else zi
    c = mesh.vertex_colors.cpu() if mesh.has_vertex_colors() else None
    return v, c, t


def check_mesh(vol, ref):
    mesh = vol.extract_triangle_mesh()
    v, c, t = arrays(mesh)
    rv, rc, rt = M.extract_triangle_mesh(ref)
    assert same(v, rv) and same(t, rt)
    assert (c is None and (rc is None or len(rc) == 0)) or same(c, rc)
    if len(rt):
        assert same(mesh.compute_triangle_normals(True).triangle_normals.cpu(), M.triangle_normals(rv, rt, True))
        mesh.triangle_normals = None
        mesh.compute_vertex_normals()
        rvn, rtn = M.compute_vertex_normals(rv, rt)
        assert same(mesh.vertex_normals.cpu(), rvn) and same(mesh.triangle_normals.cpu(), rtn)
    return len(rv), len(rt)


def write_planes(vol, ref):
    """the oracle volume's host planes into the device volume, through cphb_tsdf_data"""
    import torch
    tw, col = vol.planes()
    torch.as_tensor(tw, device="cuda").copy_(torch.from_numpy(ref.tw))
    if col is not None:
        torch.as_tensor(col, device="cuda").copy_(torch.from_numpy(ref.col))
    torch.cuda.synchronize()


def intrinsic(K, w, h):
    K = np.asarray(K, np.float32)
    return CAM.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])


def test_real_frames_match_oracle():
    g = np.load(GOLDEN)
    K = CAM.PinholeCameraIntrinsic(CAM.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    vol = I.UniformTSDFVolume(8.0, 200, 0.04, CT.RGB8)
    ref = T.Volume(8.0, 200, 0.04, T.RGB8)
    rng = np.random.default_rng(5)
    for i in range(5):
        color = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(color), G.Image(g["depth"][i]), 1000.0, 4.0, False)
        vol.integrate(im, K, g["extrinsics"][i])
        ref.integrate(T.depth_to_float(g["depth"][i], 1000.0, 4.0), color, K.intrinsic_matrix, g["extrinsics"][i])
    assert check_mesh(vol, ref) == (3198, 4402)


@pytest.mark.parametrize("ct", [CT.NoColor, CT.RGB8, CT.Gray32])
def test_sphere_views_match_oracle(ct):
    w, h, res = 160, 120, 128
    vol = I.UniformTSDFVolume(2.0, res, 0.06, ct, origin=(0.01, -0.02, 0.03))
    ref = T.Volume(2.0, res, 0.06, int(ct), origin=(0.01, -0.02, 0.03))
    rng = np.random.default_rng(int(ct))
    for K, E in ring_cameras(12, w, h, 2.5):
        color = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(color), G.Image(d16), 1000.0, 100.0, ct == CT.Gray32)
        vol.integrate(im, intrinsic(K, w, h), E)
        d = T.depth_to_float(d16, 1000.0, 100.0)
        ref.integrate(d, None if ct == CT.NoColor else (T.intensity(color) if ct == CT.Gray32 else color), K, E)
    nv, nt = check_mesh(vol, ref)
    assert nv > 10000 and nt > 10000


def test_all_256_single_cube_configurations():
    rng = np.random.default_rng(2)
    vol = I.UniformTSDFVolume(1.0, 2, 0.1, CT.RGB8, origin=(0.1, 0.2, -0.3))
    ref = T.Volume(1.0, 2, 0.1, T.RGB8, origin=(0.1, 0.2, -0.3))
    corner = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
    for ci in range(256):
        for i, (x, y, z) in enumerate(corner):
            m = np.float32(rng.uniform(0.01, 1.0))
            ref.tw[(x * 2 + y) * 2 + z] = (-m if ci >> i & 1 else m, 1.0)
        ref.col[:] = rng.uniform(0, 255, ref.col.shape).astype(np.float32)
        write_planes(vol, ref)
        nv, nt = check_mesh(vol, ref)
        assert (nv == 0) == (ci in (0, 255))


@pytest.mark.parametrize("ct", [CT.NoColor, CT.RGB8, CT.Gray32])
def test_random_fields_match_oracle(ct):
    rng = np.random.default_rng(10 + int(ct))
    res = 48
    vol = I.UniformTSDFVolume(2.0, res, 0.1, ct)
    ref = T.Volume(2.0, res, 0.1, int(ct))
    ref.tw[:, 0] = rng.uniform(-1, 1, res ** 3).astype(np.float32)
    ref.tw[:, 1] = (rng.random(res ** 3) > 0.05).astype(np.float32) * rng.uniform(1, 5, res ** 3).astype(np.float32)
    ref.col[:] = rng.uniform(0, 255, ref.col.shape).astype(np.float32)
    write_planes(vol, ref)
    nv, nt = check_mesh(vol, ref)
    assert nv > 50000


@pytest.fixture(scope="module")
def sphere_volume():
    w, h = 160, 120
    vol = I.UniformTSDFVolume(2.0, 128, 0.06, CT.RGB8)
    rng = np.random.default_rng(1)
    for K, E in ring_cameras(8, w, h, 2.5):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)), G.Image(d16),
                                                     1000.0, 100.0, False)
        vol.integrate(im, intrinsic(K, w, h), E)
    return vol


def test_repeats_are_bit_identical_and_the_launch_count_fixed(sphere_volume):
    a, b = arrays(sphere_volume.extract_triangle_mesh()), arrays(sphere_volume.extract_triangle_mesh())
    assert len(a[2]) > 1000 and all(same(x, y) for x, y in zip(a, b))
    L = _lib.lib()
    empty = I.UniformTSDFVolume(2.0, 128, 0.06, CT.RGB8)
    nv, nt = ctypes.c_size_t(0), ctypes.c_size_t(0)
    cap = 400000
    v, c, t = DeviceArray((cap, 3), np.float32), DeviceArray((cap, 3), np.float32), DeviceArray((cap, 3), np.int32)
    counts = []
    for args in ((None, None, None, 0, 0), (v.ptr, c.ptr, t.ptr, cap, cap)):
        for vol in (sphere_volume, empty):
            n0 = L.cphb_launch_count()
            _lib.check(L.cphb_tsdf_extract_mesh(vol._h, *args, ctypes.byref(nv), ctypes.byref(nt), None))
            counts.append(L.cphb_launch_count() - n0)
    assert len(set(counts)) == 1 and counts[0] > 0, counts


def test_empty_volume_and_reset_give_an_empty_mesh(sphere_volume):
    vol = I.UniformTSDFVolume(2.0, 64, 0.06, CT.Gray32)
    m = vol.extract_triangle_mesh()
    assert not m.has_vertices() and not m.has_triangles() and not m.has_vertex_colors()
    K, E = ring_cameras(1, 160, 120, 2.5)[0]
    d16 = np.round(sphere_depth(K, E, 160, 120, 0.6) * 1000).astype(np.uint16)
    im = G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((120, 160, 3), np.uint8)), G.Image(d16), 1000.0, 100.0, True)
    vol.integrate(im, intrinsic(K, 160, 120), E)
    assert vol.extract_triangle_mesh().has_triangles()
    vol.reset()
    m = vol.extract_triangle_mesh()
    assert not m.has_vertices() and not m.has_triangles()
    m.compute_vertex_normals()  # an empty mesh's normals are empty
    assert len(m.vertex_normals) == 0 and len(m.triangle_normals) == 0


def test_sizing_and_writing_calls_agree(sphere_volume):
    L = _lib.lib()
    nv, nt = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _lib.check(L.cphb_tsdf_extract_mesh(sphere_volume._h, None, None, None, 0, 0, ctypes.byref(nv), ctypes.byref(nt), None))
    sized = (nv.value, nt.value)
    v, c, t = arrays(sphere_volume.extract_triangle_mesh())
    assert sized == (len(v), len(t))
    # one capacity too small: the counts come back and nothing is written
    import torch
    vb = DeviceArray((sized[0], 3), np.float32)
    cb = DeviceArray((sized[0], 3), np.float32)
    tb = DeviceArray((sized[1], 3), np.int32)
    torch.as_tensor(tb, device="cuda").fill_(-7)
    _lib.check(L.cphb_tsdf_extract_mesh(sphere_volume._h, vb.ptr, cb.ptr, tb.ptr, sized[0], sized[1] - 1, ctypes.byref(nv),
                                        ctypes.byref(nt), None))
    assert (nv.value, nt.value) == sized and np.all(tb.cpu() == -7)
    with pytest.raises(_lib.CphbError):  # capacity without outputs
        _lib.check(L.cphb_tsdf_extract_mesh(sphere_volume._h, None, None, None, 10, 10, ctypes.byref(nv), ctypes.byref(nt), None))


def test_mesh_from_arrays_normals_and_index_checks():
    v = np.float32([[0, 0, 0], [1, 0, 0], [5, 5, 5], [0, 1, 0], [0, 0, 1]])
    t = np.int32([[0, 1, 3], [0, 3, 4], [0, 4, 1]])
    m = G.TriangleMesh(v, t)
    assert m.has_vertices() and m.has_triangles() and not m.has_vertex_normals()
    m.compute_vertex_normals(False)
    rvn, rtn = M.compute_vertex_normals(v, t, normalized=False)
    assert same(m.vertex_normals.cpu(), rvn) and same(m.triangle_normals.cpu(), rtn) and np.all(rvn[2] == 0)
    bad = G.TriangleMesh(v, np.int32([[0, 1, 5]]))
    with pytest.raises(_lib.CphbError):
        bad.compute_triangle_normals()
    bad.triangle_normals = np.zeros((1, 3), np.float32)
    with pytest.raises(_lib.CphbError):
        bad.compute_vertex_normals()
