"""GPU: bounding-box selection and point-cloud cleanup (csrc/crop.cu) against the CPU restatement (oracle/crop.c).

- The kept indices of the AABB, OBB, pass-through and finite tests equal the oracle's bit for bit at sizes around warp
  and block boundaries up to 1 M points, and on the 10 M config-3 cloud with 1 % NaN / inf rows.
- OrientedBoundingBox::CreateFromPoints (centre, R, extent), UniformDownSample and both normal operations equal the
  oracle bit for bit; the reference's known answers hold on the device.
- The Python methods carry normals and colours row for row, handle covariances as the reference does, handle bad
  arguments and degenerate clouds, repeat bit for bit, and a crop launches the flag kernel, the shared compaction and
  the gather and nothing else."""
import json
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing import datagen

G = cph.geometry
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [0, 1, 31, 32, 33, 1023, 1024, 1025, 100_000, 1_000_000]


@pytest.fixture(scope="module")
def cp():
    from oracle import crop_py
    crop_py.build()
    return crop_py


@pytest.fixture(scope="module")
def known():
    with open(os.path.join(ROOT, "tests", "golden", "pointcloud_crop_known.json")) as f:
        return json.load(f)


def _cloud(n, seed, bad_frac=0.0):
    """config-3 shaped points (uniform in [0,4)x[0,4)x[0,1)); bad_frac of the rows get a NaN or +-inf coordinate"""
    pts = datagen.uniform_cube(n, seed, hi=(4, 4, 1))
    if bad_frac and n:
        rng = np.random.default_rng(seed + 1)
        rows = rng.choice(n, max(1, int(n * bad_frac)), replace=False)
        pts[rows, rng.integers(0, 3, len(rows))] = rng.choice(np.float32([np.nan, np.inf, -np.inf]), len(rows))
    return pts


OBB = ((2.0, 2.0, 0.5), [[0.8660254, -0.5, 0.0], [0.5, 0.8660254, 0.0], [0.0, 0.0, 1.0]], (2.6, 2.6, 1.2))


def _check_selections(cp, pts):
    d = G.PointCloud(pts).points
    lo, hi = (0.5, 1.0, 0.25), (2.0, 4.0, 0.75)
    np.testing.assert_array_equal(G.AxisAlignedBoundingBox(lo, hi).get_point_indices_within_bounding_box(d).cpu(),
                                  cp.aabb_indices(pts, lo, hi))
    obb = G.OrientedBoundingBox(*OBB)
    np.testing.assert_array_equal(obb.get_point_indices_within_bounding_box(d).cpu(),
                                  cp.obb_indices(pts, obb.get_box_points()))
    for flags in ((1, 1), (1, 0), (0, 1)):
        got = _device_finite(d, len(pts), *flags)
        np.testing.assert_array_equal(got, cp.finite_indices(pts, *flags))


def _device_finite(d, n, rm_nan, rm_inf):
    import ctypes as C
    from cupoch_b200.utility import DeviceArray
    out = DeviceArray((max(n, 1),), np.int32)
    m = C.c_size_t(0)
    _lib.check(_lib.lib().cphb_finite_point_indices(d.ptr if n else None, n, rm_nan, rm_inf, out.ptr, C.byref(m), None))
    return out.cpu()[:m.value]


@pytest.mark.parametrize("n", SIZES)
def test_indices_equal_oracle(cp, n):
    _check_selections(cp, _cloud(n, 31, bad_frac=0.01))


def test_indices_10m_with_non_finite_rows(cp):
    pts = _cloud(10_000_000, 41, bad_frac=0.01)
    _check_selections(cp, pts)
    pc = G.PointCloud(pts)
    for axis in range(3):
        np.testing.assert_array_equal(pc.pass_through_filter(axis, 0.25, 0.75).points.cpu(),
                                      pts[cp.pass_through_indices(pts, axis, 0.25, 0.75)])


@pytest.mark.parametrize("n,seed", [(1, 1), (2, 2), (33, 3), (1025, 4), (100_000, 5), (1_000_000, 6)])
def test_oriented_bounding_box_equals_oracle(cp, n, seed):
    rng = np.random.default_rng(seed)
    pts = (_cloud(n, seed) * rng.uniform(0.2, 3, 3) @ datagen.rot_xyz(10 * seed, -7, 3 * seed).T).astype(np.float32)
    obb = G.PointCloud(pts).get_oriented_bounding_box()
    c, R, e = cp.obb_create(pts)
    np.testing.assert_array_equal(obb.center, c)
    np.testing.assert_array_equal(obb.R, R)
    np.testing.assert_array_equal(obb.extent, e)


def test_oriented_bounding_box_known_answers(cp, known):
    g = known["oriented_bounding_box"]
    obb = G.PointCloud(np.float32(g["points_8"])).get_oriented_bounding_box()
    np.testing.assert_array_equal(obb.center, np.float32(g["center"]))
    np.testing.assert_array_equal(obb.extent, np.float32(g["extent"]))
    np.testing.assert_array_equal(obb.R, np.float32(g["R"]))
    bp = obb.get_box_points().astype(np.float64)
    ref = np.float64(g["box_points"])
    np.testing.assert_array_equal(bp[np.lexsort(bp.T[::-1])], ref[np.lexsort(ref.T[::-1])])
    c, R, e = cp.obb_create(g["points_4"])
    obb4 = G.PointCloud(np.float32(g["points_4"])).get_oriented_bounding_box()
    np.testing.assert_array_equal(obb4.R, R)
    np.testing.assert_array_equal(obb4.extent, e)


def test_uniform_down_sample_equals_oracle(cp, known):
    g = known["uniform_down_sample"]
    out = G.PointCloud(np.float32(g["points"])).uniform_down_sample(g["every_k_points"])
    np.testing.assert_allclose(out.points.cpu(), g["ref"], atol=known["tolerance"])
    pts = _cloud(1_000_003, 7)
    pc = G.PointCloud(pts)
    pc.normals = datagen.unit_normals(len(pts), 8)
    pc.colors = datagen.uniform_cube(len(pts), 9)
    for k in (1, 2, 5, 7, 1_000_003, 2_000_000):
        rows = cp.uniform_rows(len(pts), k)
        out = pc.uniform_down_sample(k)
        assert len(out) == len(rows)
        if len(rows):
            np.testing.assert_array_equal(out.points.cpu(), pts[rows])
            np.testing.assert_array_equal(out.normals.cpu(), pc.normals.cpu()[rows])
            np.testing.assert_array_equal(out.colors.cpu(), pc.colors.cpu()[rows])


def _odd_normals(n, seed):
    rng = np.random.default_rng(seed)
    nrm = rng.normal(size=(n, 3)).astype(np.float32) * rng.uniform(1e-3, 1e3, (n, 1)).astype(np.float32)
    nrm[::97] = 0.0
    nrm[1::97] = np.float32([0, 0, -0.0])
    nrm[2::97] = np.float32([1e-30, 0, 0])
    nrm[3::97, 0] = np.nan
    nrm[4::97] = np.float32([1, 0, 0])  # orthogonal to the reference below
    return nrm


def test_normal_operations_equal_oracle(cp, known):
    nrm = _odd_normals(300_001, 11)
    pc = G.PointCloud(np.zeros_like(nrm))
    pc.normals = nrm
    pc.normalize_normals()
    np.testing.assert_array_equal(pc.normals.cpu(), cp.normalize_normals(nrm))
    pc.normals = nrm
    assert pc.orient_normals_to_align_with_direction((0.0, 0.5, 2.0))
    np.testing.assert_array_equal(pc.normals.cpu(), cp.orient_normals(nrm, (0.0, 0.5, 2.0)))
    g = known["normalize_normals"]
    pc = G.PointCloud(np.zeros((20, 3), np.float32))
    pc.normals = np.float32(g["normals"])
    np.testing.assert_allclose(pc.normalize_normals().normals.cpu(), g["ref"], atol=known["tolerance"])
    g = known["orient_normals"]
    pc = G.PointCloud(np.float32(g["points"]))
    pc.estimate_normals(G.KDTreeSearchParamKNN(g["knn"]))
    pc.orient_normals_to_align_with_direction(g["reference"])
    np.testing.assert_allclose(pc.normals.cpu(), g["ref"], atol=known["tolerance"])


def _full_cloud(n, seed, bad_frac=0.0):
    pc = G.PointCloud(_cloud(n, seed, bad_frac))
    pc.normals = datagen.unit_normals(n, seed + 2)
    pc.colors = datagen.uniform_cube(n, seed + 3)
    pc.covariances = np.tile(np.eye(3, dtype=np.float32), (n, 1, 1))
    return pc


def test_methods_carry_attributes_row_for_row(cp):
    pc = _full_cloud(50_000, 51, bad_frac=0.02)
    pts, nrm, col = pc.points.cpu(), pc.normals.cpu(), pc.colors.cpu()
    cases = [(pc.crop(G.AxisAlignedBoundingBox((1, 1, 0), (3, 3, 1))), cp.aabb_indices(pts, (1, 1, 0), (3, 3, 1))),
             (pc.crop(G.OrientedBoundingBox(*OBB)), cp.obb_indices(pts, G.OrientedBoundingBox(*OBB).get_box_points())),
             (pc.pass_through_filter(1, 0.5, 2.5), cp.pass_through_indices(pts, 1, 0.5, 2.5))]
    for out, idx in cases:
        assert 0 < len(idx) < len(pts)
        np.testing.assert_array_equal(out.points.cpu(), pts[idx])
        np.testing.assert_array_equal(out.normals.cpu(), nrm[idx])
        np.testing.assert_array_equal(out.colors.cpu(), col[idx])
        assert not out.has_covariances()
    idx = cp.finite_indices(pts)
    assert pc.remove_none_finite_points() is pc
    np.testing.assert_array_equal(pc.points.cpu(), pts[idx])
    np.testing.assert_array_equal(pc.normals.cpu(), nrm[idx])
    np.testing.assert_array_equal(pc.colors.cpu(), col[idx])
    assert pc.has_normals() and pc.has_colors() and not pc.has_covariances()  # rows removed: covariances dropped


def test_covariances_kept_when_nothing_is_removed():
    pc = _full_cloud(1000, 61)
    pc.remove_none_finite_points()
    assert pc.has_covariances() and len(pc) == 1000
    out = pc.pass_through_filter(2, -1.0, 2.0)  # keeps every row: the reference's copy keeps the covariances
    assert len(out) == 1000 and out.has_covariances()
    np.testing.assert_array_equal(out.covariances.cpu(), pc.covariances.cpu())


def test_argument_handling(capsys):
    pc = _full_cloud(1000, 71)
    assert pc.pass_through_filter(3, 0, 1).is_empty()
    assert pc.pass_through_filter(-1, 0, 1).is_empty()
    assert "axis_no must be 0, 1 or 2" in capsys.readouterr().err
    assert pc.uniform_down_sample(0).is_empty()
    assert "Illegal sample rate" in capsys.readouterr().err
    assert len(pc.uniform_down_sample(1001)) == 0 and len(pc.uniform_down_sample(1000)) == 1
    # an empty box is logged and the crop still runs: the flat box keeps the points on its plane
    flat = G.PointCloud(np.float32([[0, 0, 0], [1, 1, 0], [1, 1, 1], [0.5, 0.5, 0]]))
    assert len(flat.crop(G.AxisAlignedBoundingBox((0, 0, 0), (1, 1, 0)))) == 3
    assert "AxisAlignedBoundingBox either has zeros size" in capsys.readouterr().err
    with pytest.raises(TypeError):
        pc.crop(((0, 0, 0), (1, 1, 1)))
    import ctypes as C
    m = C.c_size_t(7)
    assert _lib.lib().cphb_uniform_down_sample(pc.points.ptr, None, None, 1000, 0, pc.points.ptr, None, None, C.byref(m),
                                               None) == _lib.CPHB_ERR_INVALID and m.value == 0


def test_empty_and_all_nan_clouds(capsys):
    e = G.PointCloud()
    assert e.crop(G.AxisAlignedBoundingBox((0, 0, 0), (1, 1, 1))).is_empty()
    assert e.crop(G.OrientedBoundingBox(*OBB)).is_empty()
    assert e.pass_through_filter(0, 0, 1).is_empty()
    assert e.uniform_down_sample(3).is_empty()
    assert e.remove_none_finite_points().is_empty()
    obb = e.get_oriented_bounding_box()
    np.testing.assert_array_equal(obb.R, np.eye(3, dtype=np.float32))
    assert not obb.center.any() and not obb.extent.any()
    aabb = e.get_axis_aligned_bounding_box()
    assert not aabb.min_bound.any() and not aabb.max_bound.any()
    assert not e.orient_normals_to_align_with_direction()
    assert "No normals" in capsys.readouterr().err
    nan = G.PointCloud(np.full((1000, 3), np.nan, np.float32))
    assert len(nan.crop(G.AxisAlignedBoundingBox((0, 0, 0), (1, 1, 1)))) == 1000  # NaN points are kept
    assert len(nan.pass_through_filter(1, 0, 1)) == 1000
    assert nan.crop(G.OrientedBoundingBox(*OBB)).is_empty()
    nan.normals = np.ones((1000, 3), np.float32)
    assert nan.remove_none_finite_points().is_empty() and not nan.has_normals()


def test_aabb_accessors_and_box_points():
    b = G.AxisAlignedBoundingBox((1, 2, 3), (4, 6, 8))
    np.testing.assert_array_equal(b.get_center(), [2.5, 4, 5.5])
    np.testing.assert_array_equal(b.get_extent(), [3, 4, 5])
    np.testing.assert_array_equal(b.get_half_extent(), [1.5, 2, 2.5])
    assert b.get_max_extent() == 5 and b.volume() == 60 and not b.is_empty()
    bp = b.get_box_points()
    assert bp.shape == (8, 3) and {tuple(r) for r in bp.tolist()} == {(x, y, z) for x in (1, 4) for y in (2, 6) for z in (3, 8)}
    o = G.OrientedBoundingBox.create_from_axis_aligned_bounding_box(b)
    np.testing.assert_array_equal(o.get_min_bound(), b.min_bound)
    np.testing.assert_array_equal(o.get_max_bound(), b.max_bound)
    pts = _cloud(5000, 81)
    a = G.AxisAlignedBoundingBox.create_from_points(pts)
    np.testing.assert_array_equal(a.min_bound, pts.min(0))
    np.testing.assert_array_equal(a.max_bound, pts.max(0))


def test_calls_repeat_bit_for_bit():
    pc = _full_cloud(200_000, 91, bad_frac=0.01)
    obb = G.OrientedBoundingBox(*OBB)
    for f in (lambda: pc.crop(obb).points.cpu(), lambda: pc.pass_through_filter(0, 1, 3).colors.cpu(),
              lambda: pc.uniform_down_sample(3).normals.cpu(),
              lambda: np.concatenate([x.reshape(-1) for x in (lambda o: (o.center, o.R, o.extent))(
                  G.PointCloud(pc.points.cpu()[np.isfinite(pc.points.cpu()).all(1)]).get_oriented_bounding_box())])):
        a, b = f(), f()
        assert a.tobytes() == b.tobytes()


_LAUNCH_LIST_SCRIPT = r"""
import sys
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import torch
from torch.profiler import ProfilerActivity, profile
import test_gpu_crop as t
pc = t._full_cloud(100_000, 101)
box = t.G.AxisAlignedBoundingBox((0, 0, 0), (2, 4, 1))
pc.crop(box)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    pc.crop(box)
    torch.cuda.synchronize()
for e in prof.key_averages():
    if "CUDA" in str(getattr(e, "device_type", "")) and "Memset" not in e.key and "Memcpy" not in e.key:
        print("KERNEL", e.key)
"""


def test_crop_launch_list():
    """a crop is the flag kernel, the shared compaction's three kernels and the gather: five launches, named so in
    torch.profiler.  The profiled call runs in a child process, so that this process's later profiler sessions (other
    test files use torch.profiler too) start from a fresh profiler state."""
    import subprocess
    import sys
    L = _lib.lib()
    pc = _full_cloud(100_000, 101)
    box = G.AxisAlignedBoundingBox((0, 0, 0), (2, 4, 1))
    pc.crop(box)
    before = L.cphb_launch_count()
    pc.crop(box)
    assert L.cphb_launch_count() - before == 5
    r = subprocess.run([sys.executable, "-c", _LAUNCH_LIST_SCRIPT % (ROOT, os.path.join(ROOT, "tests"))], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    names = sorted({ln[len("KERNEL "):] for ln in r.stdout.splitlines() if ln.startswith("KERNEL ")})
    expect = ["crop_flag_kernel", "keep_count_kernel", "keep_scan_kernel", "keep_write_kernel", "select_rows_kernel"]
    assert len(names) == len(expect), names
    for k in expect:
        assert sum(k in nm for nm in names) == 1, (k, names)
