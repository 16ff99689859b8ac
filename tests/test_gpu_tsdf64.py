"""GPU: ExtractPointCloud and Raycast of csrc/tsdf.cu on the cases of test_oracle_tsdf64.py, held both to oracle/tsdf.c
bit for bit and, directly, to the float64 restatement (cupoch_b200/testing/tsdf64.py) and the analytic planar and
spherical fields, so the device evidence does not rest on the oracle alone.  Also the sphere-view comparison of every
extractor, ExtractTriangleMesh included, at odd resolutions, and the largest grid the volume allows (res 1290, whose
res^3 just fits the int32 positions of the compaction) with a field written into a slab at its far corner."""
import time
import types

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200.testing import tsdf64 as X
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import tsdf_mesh_py as M, tsdf_py as T
from test_gpu_tsdf import check_extractions, check_raycast, cloud, intrinsic, oracle_frame, rgbd, same
from test_gpu_tsdf_mesh import check_mesh, write_planes
from test_oracle_tsdf64 import (NORMALS, axis_camera, axis_rays, check_points, check_rays, look_at, odd_volume, plane_case,
                                plane_sdf, six_faces_inside_and_on_the_box, sphere_sdf, within, written)

I = cph.integration
CT = I.TSDFVolumeColorType
U = X.EPS32


def device_of(ref):
    vol = I.UniformTSDFVolume(ref.length, ref.res, ref.trunc, CT(ref.ct), origin=tuple(ref.origin))
    write_planes(vol, ref)
    return vol


def same_points(vol, ref):
    """the device extraction equals the oracle's bit for bit and meets the float64 checks -> the device rows"""
    p, n, c = cloud(vol.extract_point_cloud())
    rp, rn, rc = ref.extract_point_cloud()
    assert same(p, rp) and same(n, rn) and same(c, rc if rc is not None else np.zeros((0, 3), np.float32))
    check_points(ref, p, n, c if ref.ct != T.NO_COLOR else None)
    return p, n


def same_rays(vol, ref, K, E, w, h, trunc, **kw):
    """the device raycast (one row per pixel) equals the oracle's bit for bit and meets the float64 checks"""
    rows = cloud(vol.raycast(intrinsic(K, w, h), E, trunc, False))
    want = ref.raycast(K, E, w, h, trunc, False)
    assert all(same(a, b) for a, b in zip(rows, want))
    ray, _, _ = check_rays(ref, K, E, w, h, trunc, rows, **kw)
    return rows, ray


# ------------------------------------------------------------------------------------------------ the CPU cases
@pytest.mark.parametrize("ckind", ["random", "centre", "face"])
@pytest.mark.parametrize("nkind", list(NORMALS))
def test_planar_fields(nkind, ckind):
    ref, n, c = plane_case(nkind, ckind)
    vol = device_of(ref)
    p, nrm = same_points(vol, ref)
    if len(p):
        assert within(p, plane_sdf(n, c), 4 * U * 2 * ref.length) and np.all(np.abs(nrm - n) <= 64 * U * ref.res)
    vl, trunc, w, h = float(ref.voxel_length), float(ref.trunc), 48, 36
    side = np.cross(n, [0.3, 0.5, 0.8])
    rows, _ = same_rays(vol, ref, *look_at(2.5 * n + 0.2 * side, -0.3 * side, w, h, 30.0), w, h, trunc)
    hit = np.isfinite(rows[0][:, 0])
    assert within(rows[0][hit], plane_sdf(n, c), 0.5 * np.abs(n).sum() * vl + 32 * U)
    assert np.all(np.abs(rows[1][hit] - n) <= 64 * U * ref.res)
    rows, _ = same_rays(vol, ref, *look_at(-2.5 * n + 0.2 * side, -0.3 * side, w, h, 30.0), w, h, trunc)
    assert not np.isfinite(rows[0][:, 0]).any()


@pytest.mark.parametrize("res", [3, 5, 63, 64, 65, 129])
def test_written_spheres_and_odd_resolutions(res):
    ref = odd_volume(res)
    vol = device_of(ref)
    p, n = same_points(vol, ref)
    vl = float(ref.voxel_length)
    if res >= 63:
        assert within(p, sphere_sdf(0.6), np.sqrt(3) / 2 * vl + vl * vl / 0.6)
    for K, E in ring_cameras(3, 40, 30):
        rows, ray = same_rays(vol, ref, K, E, 40, 30, float(ref.trunc))
        hit = np.isfinite(rows[0][:, 0])
        if res == 3:
            assert not hit.any()
        if res >= 63:
            assert within(rows[0][hit], sphere_sdf(0.6), np.sqrt(3) / 2 * vl + vl * vl / 0.6)


def test_cameras_faces_inside_on_the_box_grazing_and_axis_rays():
    ref = odd_volume(63)
    vol = device_of(ref)
    for name, K, E in six_faces_inside_and_on_the_box(ref):
        _, ray = same_rays(vol, ref, K, E, 40, 30, float(ref.trunc))
        assert (not ray.hit.any()) if name == "inside sphere" else ray.hit.sum() > 100, name
    vl = float(ref.voxel_length)
    o = ref.origin.astype(np.float64)
    lo, hi = -(63 // 2) * vl, (63 - 1 - 63 // 2) * vl
    for target in ([lo, lo, 0.0], [lo, hi, 0.2], [lo, lo, lo], [hi, hi, hi]):
        t = np.asarray(target) + o
        same_rays(vol, ref, *look_at([t[0] - 2.0, t[1] - 1.0, t[2] + 0.5], t, 9, 9, 8.0), 9, 9, float(ref.trunc), max_listed=9)
    # axis-parallel rays along cell faces: every decision exact, no slack
    ref2 = written(32, 2.0, 0.125, sphere_sdf(0.6))
    vol2 = device_of(ref2)
    hits = 0
    for K, E in axis_rays():
        rows, ray = same_rays(vol2, ref2, K, E, 1, 1, 0.125, max_listed=1)
        assert np.isfinite(rows[0][0, 0]) == ray.hit[0]
        if ray.hit[0]:
            hits += 1
            assert np.array_equal(np.round(rows[2][0] * 255).astype(np.int64), ray.voxel[0])
    assert hits >= 50
    # len + step == len at entry: a miss on the device as in the oracle, where float64 hits
    K, E = axis_camera([-3.0e6, 0.0, 0.0], 0, 1)
    rows, ray = same_rays(vol2, ref2, K, E, 1, 1, 0.04, max_listed=1)
    assert not np.isfinite(rows[0][0, 0]) and ray.hit[0]


@pytest.mark.parametrize("ray_trunc", [0.04, 0.5])
def test_short_steps_and_a_thin_shell(ray_trunc):
    shell = lambda x: np.abs(np.linalg.norm(x, axis=-1) - 0.6) - 0.0317  # noqa: E731
    ref = written(63, 2.0, 0.06, shell if ray_trunc > 0.1 else sphere_sdf(0.6), origin=(0.0123, -0.0311, 0.0057))
    vol = device_of(ref)
    for K, E in ring_cameras(2, 48, 36):
        same_rays(vol, ref, K, E, 48, 36, ray_trunc)


# ------------------------------------------------------------------------------------------------ odd-res sphere views
@pytest.mark.parametrize("res", [5, 63, 129])
def test_odd_res_sphere_views_match_oracle_for_every_extractor(res):
    w, h, length, trunc = 160, 120, 2.0, max(0.06, 2.5 * 2.0 / res)
    ct = CT.RGB8
    vol = I.UniformTSDFVolume(length, res, trunc, ct, origin=(0.0123, -0.0311, 0.0057))
    ref = T.Volume(length, res, trunc, int(ct), origin=(0.0123, -0.0311, 0.0057))
    rng = np.random.default_rng(res)
    cams = ring_cameras(8, w, h, 2.5)
    for K, E in cams:
        color = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        im, d16 = rgbd(sphere_depth(K, E, w, h, 0.6), color, ct)
        vol.integrate(im, intrinsic(K, w, h), E)
        ref.integrate(*oracle_frame(d16, color, ct), K, E)
    npts, nvox = check_extractions(vol, ref)
    nv, nt = check_mesh(vol, ref)
    rays = sum(check_raycast(vol, ref, K, E, w, h, trunc) for K, E in cams[:2])
    if res >= 63:
        assert npts > 1000 and nvox > 1000 and nt > 1000 and rays > 1000
        check_points(ref)


# ------------------------------------------------------------------------------------------------ the largest grid
RES_MAX = 1290


@pytest.fixture
def pool_released():
    """after the test, hand the device's default memory pool's free blocks back to the driver: the library keeps freed
    blocks for reuse, and the largest grid's 47 GB would otherwise stay reserved for the rest of the session"""
    yield
    import ctypes
    import gc
    import torch
    gc.collect()
    torch.cuda.synchronize()
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool = ctypes.c_int(), ctypes.c_void_p()
    assert cu.cuCtxGetDevice(ctypes.byref(dev)) == 0
    assert cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    assert cu.cuMemPoolTrimTo(pool, ctypes.c_size_t(0)) == 0


def test_largest_grid_slab_at_the_far_corner(pool_released):
    """res 1290 (res^3 = 2,146,689,000 voxels, below 2^31 - 1), NoColor, vl = 1 / 64.  A planar field is written into
    the 25^3 voxels [1265, 1290)^3 only, through a slice of the device plane; nothing else is copied to or from the host.
    The counts of ExtractPointCloud, ExtractVoxelPointCloud and ExtractTriangleMesh and a raycast aimed at the slab are
    held to tsdf64 (and the mesh oracle) run on the 26^3 block [1264, 1290)^3 alone.
    Memory by arithmetic: the volume 8 B a voxel (17.2 GB); ExtractTriangleMesh's scratch, the largest, 14 B a voxel
    (two byte planes and three int32 position planes, 30.1 GB): 22 B a voxel, 47.2 GB in all."""
    import torch
    res = RES_MAX
    n = res ** 3
    need = 22 * n + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB are free" % (need / 1e9, free / 1e9))
    length, vl = res / 64.0, 1.0 / 64.0
    trunc = 5 * vl
    k0, S = res - 26, 26
    origin = (0.25, -0.5, 0.125)
    o = np.asarray(origin, np.float64)
    h = res // 2
    normal = np.array([0.31, -0.72, 0.55])
    normal /= np.linalg.norm(normal)
    mid = (k0 + 13 - h + 0.5) * vl + o
    c = float(normal @ mid) + 0.3 * vl
    k = np.arange(k0, res)
    cen = np.stack(np.meshgrid(*[(k - h + 0.5) * vl + o[a] for a in range(3)], indexing="ij"), -1)
    block = np.zeros((S, S, S, 2), np.float32)
    block[1:, 1:, 1:, 0] = np.clip((cen[1:, 1:, 1:] @ normal - c) / np.float32(trunc), -1, 1)
    block[1:, 1:, 1:, 1] = 1.0
    timings = {}
    t0 = time.perf_counter()
    vol = I.UniformTSDFVolume(length, res, trunc, CT.NoColor, origin=origin)
    torch.cuda.synchronize()
    timings["create"] = time.perf_counter() - t0
    used = {"create": free - torch.cuda.mem_get_info()[0]}
    tw, _ = vol.planes()
    dev = torch.as_tensor(tw, device="cuda").view(res, res, res, 2)
    dev[k0:, k0:, k0:] = torch.from_numpy(block).cuda()
    torch.cuda.synchronize()
    del dev
    bt = block.reshape(-1, 2)
    ref = types.SimpleNamespace(tw=bt, col=None, length=length, res=res, origin=np.float32(origin), ct=T.NO_COLOR,
                                voxel_length=np.float32(vl), trunc=np.float32(trunc), block=(k0, S))

    t0 = time.perf_counter()
    p, nrm, _ = cloud(vol.extract_point_cloud(), False)
    timings["extract_point_cloud"] = time.perf_counter() - t0
    used["extract_point_cloud"] = free - torch.cuda.mem_get_info()[0]
    r = X.extract_point_cloud64(bt, None, length, res, origin, 0, block=(k0, S))
    assert len(p) == len(r.rows) > 500
    assert np.all(np.abs(p - r.points) <= 4 * U * (2 * length + 1))
    assert np.all(np.abs(nrm - r.normals) <= U * (16 * res + 64) / r.nscale[:, None])
    assert within(p, plane_sdf(normal, c), 4 * U * (2 * length + 1))

    t0 = time.perf_counter()
    vp, _, _ = cloud(vol.extract_voxel_point_cloud())
    timings["extract_voxel_point_cloud"] = time.perf_counter() - t0
    used["extract_voxel_point_cloud"] = free - torch.cuda.mem_get_info()[0]
    band = (bt[:, 1] != 0) & (bt[:, 0] < np.float32(0.98)) & (bt[:, 0] >= np.float32(-0.98))
    assert len(vp) == int(band.sum()) > 500
    want = cen.reshape(-1, 3)[band]
    assert np.all(np.abs(vp - want) <= 4 * U * (length + 1))

    t0 = time.perf_counter()
    mesh = vol.extract_triangle_mesh()
    timings["extract_triangle_mesh"] = time.perf_counter() - t0
    used["extract_triangle_mesh"] = free - torch.cuda.mem_get_info()[0]
    sub = T.Volume(S * vl, S, trunc, T.NO_COLOR, origin=tuple(o + (k0 - h + S // 2) * vl))
    sub.tw[:] = bt
    sv, _, st = M.extract_triangle_mesh(sub)
    mv = mesh.vertices.cpu()
    assert len(mv) == len(sv) > 500 and len(mesh.triangles) == len(st)
    assert np.all(np.abs(mv - sv) <= 8 * U * (length + 1))
    del mesh

    w = hh = 32
    K, E = look_at(mid + 3.0 * normal, mid, w, hh, 480.0)
    t0 = time.perf_counter()
    rows = cloud(vol.raycast(intrinsic(K, w, hh), E, trunc, False))
    timings["raycast"] = time.perf_counter() - t0
    # the slack grows with |t| / vl (about 5e-4 voxels here, 13 m from the origin at vl = 1 / 64), so more rows fall
    # under it than near the origin: up to 5 % may be listed
    ray, _, _ = check_rays(ref, K, E, w, hh, trunc, rows, max_listed=0.05 * w * hh)
    hit = np.isfinite(rows[0][:, 0])
    assert hit.sum() > 0.9 * w * hh
    assert within(rows[0][hit], plane_sdf(normal, c), 0.5 * np.abs(normal).sum() * vl + 1e-5)
    print("res 1290: seconds %s; device memory in use after each call (the pool keeps freed blocks: its high-water "
          "mark), GB %s, of %.1f GB free before" % ({k: round(v, 3) for k, v in timings.items()},
                                                    {k: round(v / 1e9, 2) for k, v in used.items()}, free / 1e9))
