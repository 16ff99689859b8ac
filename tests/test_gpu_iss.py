"""GPU: geometry::keypoint::ComputeISSKeypoints (csrc/iss.cu).

- The device equals the CPU oracle (oracle/iss.c) bit for bit: saliency bits, mask, keypoint indices and the radii used,
  from 1 point to 1 M and on a 10 M surface, with automatic and explicit radii, for max_neighbors in {0, 1, 5, 30, 100,
  256}, and on the quirk clouds of tests/test_oracle_iss.py.
- Through the Python function: normals and colours are gathered row for row, the empty and illegal-argument results,
  the radii diagnostics; two calls give identical bits.
- Every search of one call runs on one index build, and no search writes an [n][k] table: a call launches the index
  build's kernels plus exactly the fused kernels and the compaction."""
import ctypes as C

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing import datagen
from cupoch_b200.utility import DeviceArray
from test_oracle_iss import _cluster, box_lattice


@pytest.fixture(scope="module")
def isso():
    from oracle import iss_py
    iss_py.build()
    return iss_py


def device_iss(pts, salient_radius=0.0, non_max_radius=0.0, gamma_21=0.975, gamma_32=0.975, min_neighbors=5,
               max_neighbors=100, pc=None):
    """the ABI call -> (mask [n] bool, saliency [n] float32, keypoint indices, radii float32[2])"""
    pc = pc or cph.geometry.PointCloud(pts)
    n = len(pc)
    mask, idx, sal = DeviceArray((n,), np.uint8), DeviceArray((n,), np.int32), DeviceArray((n,), np.float32)
    m, radii = C.c_size_t(0), (C.c_float * 2)()
    _lib.check(_lib.lib().cphb_compute_iss_keypoints(pc.points.ptr, n, salient_radius, non_max_radius, gamma_21, gamma_32,
                                                     min_neighbors, max_neighbors, mask.ptr, idx.ptr, C.byref(m), sal.ptr,
                                                     radii, None))
    return mask.cpu().astype(bool), sal.cpu(), idx.cpu()[:m.value], np.array(radii, np.float32)


def check_oracle(isso, pts, *args, **kw):
    mask, sal, idx, radii = device_iss(pts, *args, **kw)
    o_mask, o_sal, o_radii = isso.iss_keypoints(pts, *args, **kw)
    np.testing.assert_array_equal(radii.view(np.uint32), o_radii.view(np.uint32))
    np.testing.assert_array_equal(sal.view(np.uint32), o_sal.view(np.uint32))
    np.testing.assert_array_equal(mask, o_mask)
    np.testing.assert_array_equal(idx, np.flatnonzero(o_mask))
    return mask, sal


@pytest.mark.parametrize("n", [1, 2, 5, 31, 32, 33, 1023, 1025, 100_000, 1_000_000])
def test_equals_oracle_automatic_radii(isso, n):
    pts = datagen.surface(n, 50 + n % 89)[0]
    mask, _ = check_oracle(isso, pts)
    if 1023 <= n <= 100_000:
        assert mask.any()
    if n == 1_000_000:  # 1 M points on the unit square: every covariance is within 1e-5 of zero (isZero is absolute)
        assert not mask.any()


@pytest.mark.parametrize("n", [5, 33, 1025, 100_000])
def test_equals_oracle_explicit_radii(isso, n):
    pts = datagen.surface(n, 7 + n % 13)[0]
    check_oracle(isso, pts, 0.06, 0.04)
    check_oracle(isso, pts, -0.05, 0.03, min_neighbors=0)  # a negative radius acts as |r|


@pytest.mark.parametrize("k", [0, 1, 5, 30, 100, 256])
def test_equals_oracle_max_neighbors(isso, k):
    pts = datagen.surface(30_000, 17)[0]
    check_oracle(isso, pts, max_neighbors=k)
    check_oracle(isso, pts, 0.05, 0.05, min_neighbors=min(k, 5), max_neighbors=k)


def test_10m_surface(isso):
    pts = datagen.surface(10_000_000, 29, extent=10.0)[0]  # 1e5 points per unit square: covariances above isZero's 1e-5
    mask, _ = check_oracle(isso, pts)
    assert mask.any()


def test_quirk_clouds(isso):
    P = box_lattice(16)
    check_oracle(isso, P)                                   # known answer: corners
    check_oracle(isso, P * np.float32(1e-3))                # isZero is absolute: nothing
    check_oracle(isso, np.concatenate([P, P]), 0.375, 0.25, max_neighbors=256)  # duplicates: both kept
    check_oracle(isso, np.full((500, 3), 0.25, np.float32))  # coincident points: radii 0, nothing
    c, s = np.cos(0.6), np.sin(0.6)
    R = np.array([[1, 0, 0], [0, c, -s], [0, s, c]]) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    pair = np.concatenate([_cluster((0, 0, 0), (0.10, 0.09, 0.08), R), _cluster((1, 0, 0), (0.20, 0.16, 0.13), R)])
    mask, _ = check_oracle(isso, pair, 0.25, 1.5, min_neighbors=7)  # normalised saliency decides
    assert mask[:7].all() and not mask[7:].any()
    pts = datagen.surface(4000, 6)[0]
    for k in (8, 100):  # the cap truncates the suppression window
        check_oracle(isso, pts, 0.05, 0.05, max_neighbors=k)
    for mn in (20, 21, 22):
        check_oracle(isso, pts, 0.04, 0.04, min_neighbors=mn)
    for given in ((0.2, 0.0), (0.0, 0.2)):  # both radii replaced
        check_oracle(isso, pts, *given)


def test_python_function_gathers_rows(isso):
    pts, nrm = datagen.surface(50_000, 31)
    col = datagen.texture(pts, 3)
    pc = cph.geometry.PointCloud(pts)
    pc.normals, pc.colors = nrm, col
    out, mask = cph.geometry.keypoint.compute_iss_keypoints(pc)
    o_mask, _, o_radii = isso.iss_keypoints(pts)
    assert o_mask.sum() > 0 and mask.dtype == np.bool_ and mask.shape == (len(pts),)
    np.testing.assert_array_equal(mask.cpu(), o_mask)
    np.testing.assert_array_equal(out.points.cpu(), pts[o_mask])
    np.testing.assert_array_equal(out.normals.cpu(), nrm[o_mask])
    np.testing.assert_array_equal(out.colors.cpu(), col[o_mask])
    assert pc.last_iss_radii == tuple(float(r) for r in o_radii)
    out2, _ = cph.geometry.keypoint.compute_iss_keypoints(pc, 0.05, 0.03, 0.9, 0.9, 10, max_neighbots=50)
    np.testing.assert_array_equal(out2.points.cpu(), pts[isso.iss_keypoints(pts, 0.05, 0.03, 0.9, 0.9, 10, 50)[0]])
    assert pc.last_iss_radii == (float(np.float32(0.05)), float(np.float32(0.03)))


def test_python_empty_and_illegal(capsys):
    out, mask = cph.geometry.keypoint.compute_iss_keypoints(cph.geometry.PointCloud())
    assert len(out) == 0 and len(mask) == 0
    assert "Input PointCloud is empty" in capsys.readouterr().err
    pc = cph.geometry.PointCloud(datagen.surface(1000, 2)[0])
    for bad in (-1, 257):
        out, mask = cph.geometry.keypoint.compute_iss_keypoints(pc, max_neighbots=bad)
        assert len(out) == 0 and len(mask) == 0
        assert "max_neighbors" in capsys.readouterr().err
    out, mask = cph.geometry.keypoint.compute_iss_keypoints(pc, max_neighbots=0)
    assert len(out) == 0 and mask.shape == (1000,) and not mask.cpu().any()
    few, mask = cph.geometry.keypoint.compute_iss_keypoints(cph.geometry.PointCloud(datagen.surface(4, 2)[0]))
    assert len(few) == 0 and not mask.cpu().any()


def test_abi_arguments():
    L = _lib.lib()
    pc = cph.geometry.PointCloud(datagen.surface(100, 3)[0])
    mask, m = DeviceArray((100,), np.uint8), C.c_size_t(7)
    for k in (-1, 257):  # CPHB_ERR_INVALID
        assert L.cphb_compute_iss_keypoints(pc.points.ptr, 100, 0.0, 0.0, 0.975, 0.975, 5, k, mask.ptr, None, C.byref(m),
                                            None, None, None) == -1
    radii = (C.c_float * 2)()
    assert L.cphb_compute_iss_keypoints(None, 0, 0.5, 0.25, 0.975, 0.975, 5, 100, None, None, C.byref(m), None, radii,
                                        None) == 0
    assert m.value == 0 and list(radii) == [0.5, 0.25]


def test_repeatable():
    pc = cph.geometry.PointCloud(datagen.surface(1_000_000, 8, extent=3.0)[0])
    a, b = device_iss(None, pc=pc), device_iss(None, pc=pc)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x.view(np.uint8), y.view(np.uint8))


def test_one_index_build_and_no_table():
    """a call = the index build + (kNN-2 + tile sums + radii, automatic radii only) + saliency + suppression + the
    3-kernel compaction: one index serves every search, and each search is fused into its consumer"""
    L = _lib.lib()
    pts = datagen.surface(200_000, 4)[0]
    pc = cph.geometry.PointCloud(pts)
    device_iss(None, pc=pc)  # warm-up
    before = L.cphb_launch_count()
    h = C.c_void_p()
    _lib.check(L.cphb_index_create(pc.points.ptr, len(pc), None, C.byref(h)))
    L.cphb_stream_synchronize(None)
    L.cphb_index_destroy(h)
    build = L.cphb_launch_count() - before
    assert build > 0
    for radii, extra in (((0.05, 0.03), 0), ((0.0, 0.0), 3)):
        before = L.cphb_launch_count()
        device_iss(None, *radii, pc=pc)
        assert L.cphb_launch_count() - before == build + extra + 2 + 3
