"""GPU: registration::ComputeSHOTFeature (csrc/shot.cu).

- The device equals the CPU oracle (oracle/shot.c) bit for bit on every float of every row: from 1 point to 1 M, for KNN
  k in {1, 5, 30, 100}, for radius searches with max_nn in {0, 1, 100, 256}, with the descriptor radius equal to and
  different from the search radius, on the quirk clouds of tests/test_oracle_shot.py and on a planar lattice (frame
  coordinates exactly on sector boundaries).
- Through the Python function: FeatureSHOT rows, the empty input, missing normals and illegal parameters; the C-ABI
  argument checks; two calls give identical bits.
- A call launches one index build plus the SHOT kernel, and nothing that writes an [n][k] table."""
import ctypes as C

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing import datagen
from cupoch_b200.utility import DeviceArray
from test_oracle_shot import SPACING, quirk_clouds, planar_lattice


@pytest.fixture(scope="module")
def shoto():
    from oracle import shot_py
    shot_py.build()
    return shot_py


def cloud(n, seed):
    """datagen.surface at 1e5 points per unit square"""
    return datagen.surface(n, seed, extent=float(np.sqrt(max(n, 1) / 1e5)))


def device_shot(pts, nrm, radius, knn=0, search_radius=0.0, max_nn=0):
    pc = cph.geometry.PointCloud(pts)
    pc.normals = nrm
    n = len(pc)
    out = DeviceArray((max(n, 1), 352), np.float32)
    _lib.check(_lib.lib().cphb_compute_shot_feature(pc.points.ptr, pc.normals.ptr, n, radius, knn, search_radius, max_nn,
                                                    out.ptr, None))
    return out.cpu()[:n]


def check_oracle(shoto, pts, nrm, radius, knn=0, search_radius=0.0, max_nn=0):
    got = device_shot(pts, nrm, radius, knn, search_radius, max_nn)
    want = shoto.compute_shot_feature(pts, nrm, radius, knn, search_radius, max_nn)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    return got


R = float(np.float32(5 * SPACING))


@pytest.mark.parametrize("n", [1, 2, 5, 6, 31, 32, 33, 1025, 100_000, 1_000_000])
def test_equals_oracle_sizes(shoto, n):
    pts, nrm = cloud(n, 40 + n % 97)
    f = check_oracle(shoto, pts, nrm, R, 0, R, 100)
    if n >= 1025:
        assert (np.abs(f).sum(1) > 0).mean() > 0.95


@pytest.mark.parametrize("k", [1, 5, 30, 100])
def test_equals_oracle_knn(shoto, k):
    pts, nrm = cloud(30_000, 11)
    f = check_oracle(shoto, pts, nrm, R, k)
    assert (np.abs(f).sum(1) > 0).any() == (k >= 6)
    check_oracle(shoto, pts, nrm, 0.5 * R, k)  # neighbours beyond the descriptor radius


@pytest.mark.parametrize("max_nn", [0, 1, 100, 256])
def test_equals_oracle_radius(shoto, max_nn):
    pts, nrm = cloud(30_000, 12)
    check_oracle(shoto, pts, nrm, R, 0, R, max_nn)
    check_oracle(shoto, pts, nrm, R, 0, 1.6 * R, max_nn)   # search wider than the descriptor radius
    check_oracle(shoto, pts, nrm, 1.3 * R, 0, R, max_nn)   # descriptor radius wider than the search


def test_quirk_clouds(shoto):
    for name, (pts, nrm, radius, search) in quirk_clouds().items():
        check_oracle(shoto, pts, nrm, radius, *search)


def test_planar_lattice(shoto):
    pts, nrm = planar_lattice(40)
    for search in ((0, 2.5, 100), (0, 3.2, 256), (30, 0.0, 0)):
        f = check_oracle(shoto, pts, nrm, 2.5, *search)
        assert (np.abs(f).sum(1) > 0).all()


def test_python_function(shoto):
    pts, nrm = cloud(50_000, 31)
    pc = cph.geometry.PointCloud(pts)
    pc.normals = nrm
    f = cph.registration.compute_shot_feature(pc, R, cph.geometry.KDTreeSearchParamRadius(R, 100))
    assert isinstance(f, cph.registration.FeatureSHOT) and f.dimension() == 352 and f.num() == len(pts)
    np.testing.assert_array_equal(f.cpu().view(np.uint32),
                                  shoto.compute_shot_feature(pts, nrm, R, 0, R, 100).view(np.uint32))
    g = cph.registration.compute_shot_feature(input=pc, radius=R, search_param=cph.geometry.KDTreeSearchParamKNN(30))
    np.testing.assert_array_equal(g.cpu().view(np.uint32), shoto.compute_shot_feature(pts, nrm, R, 30).view(np.uint32))


def test_python_empty_and_illegal():
    e = cph.registration.compute_shot_feature(cph.geometry.PointCloud(), 0.1, cph.geometry.KDTreeSearchParamKNN(30))
    assert e.num() == 0 and e.dimension() == 352
    pc = cph.geometry.PointCloud(datagen.surface(1000, 2)[0])
    with pytest.raises(RuntimeError, match="ComputeSHOTFeature"):
        cph.registration.compute_shot_feature(pc, 0.1, cph.geometry.KDTreeSearchParamKNN(30))
    pc.normals = datagen.surface(1000, 2)[1]
    with pytest.raises(RuntimeError, match="Unsupport search param type"):
        cph.registration.compute_shot_feature(pc, 0.1, object())
    for bad in (cph.geometry.KDTreeSearchParamKNN(101), cph.geometry.KDTreeSearchParamRadius(0.1, 257),
                cph.geometry.KDTreeSearchParamRadius(0.1, -1)):
        with pytest.raises(Exception):
            cph.registration.compute_shot_feature(pc, 0.1, bad)


def test_abi_arguments():
    L = _lib.lib()
    pts, nrm = datagen.surface(100, 3)
    pc = cph.geometry.PointCloud(pts)
    pc.normals = nrm
    out = DeviceArray((100, 352), np.float32)
    assert L.cphb_compute_shot_feature(None, None, 0, 0.1, 30, 0.0, 0, None, None) == 0
    assert L.cphb_compute_shot_feature(None, pc.normals.ptr, 100, 0.1, 30, 0.0, 0, out.ptr, None) == -1
    assert L.cphb_compute_shot_feature(pc.points.ptr, None, 100, 0.1, 30, 0.0, 0, out.ptr, None) == -1
    assert L.cphb_compute_shot_feature(pc.points.ptr, pc.normals.ptr, 100, 0.1, 30, 0.0, 0, None, None) == -1
    for knn, max_nn in ((101, 0), (0, 257), (0, -1)):
        assert L.cphb_compute_shot_feature(pc.points.ptr, pc.normals.ptr, 100, 0.1, knn, 0.1, max_nn, out.ptr, None) == -1
    assert L.cphb_compute_shot_feature(pc.points.ptr, pc.normals.ptr, 100, 0.1, 100, 0.0, 0, out.ptr, None) == 0
    assert L.cphb_compute_shot_feature(pc.points.ptr, pc.normals.ptr, 100, 0.1, 0, 0.1, 256, out.ptr, None) == 0


def test_repeatable():
    pts, nrm = cloud(1_000_000, 8)
    a, b = device_shot(pts, nrm, R, 0, R, 100), device_shot(pts, nrm, R, 0, R, 100)
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


def test_one_index_build_and_no_table():
    """a call = the index build + the SHOT kernel; the profiler sees no search kernel writing an [n][k] table"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    L = _lib.lib()
    pts, nrm = cloud(200_000, 4)
    pc = cph.geometry.PointCloud(pts)
    pc.normals = nrm
    param = cph.geometry.KDTreeSearchParamRadius(R, 100)
    cph.registration.compute_shot_feature(pc, R, param)  # warm-up
    before = L.cphb_launch_count()
    h = C.c_void_p()
    _lib.check(L.cphb_index_create(pc.points.ptr, len(pc), None, C.byref(h)))
    L.cphb_stream_synchronize(None)
    L.cphb_index_destroy(h)
    build = L.cphb_launch_count() - before
    assert build > 0
    before = L.cphb_launch_count()
    cph.registration.compute_shot_feature(pc, R, param)
    assert L.cphb_launch_count() - before == build + 1
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cph.registration.compute_shot_feature(pc, R, param)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    assert sum("shot_kernel" in k for k in names) == 1, names
    assert not any("searchk_kernel" in k or "search1_kernel" in k for k in names), names
