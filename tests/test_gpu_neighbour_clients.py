"""GPU: the launch structure of the index clients that read a neighbour table (FPFH, the colour gradient, the Gaussian,
radius and statistical filters, DBSCAN, two-pass EstimateNormals).  A call launches one index build, the standalone
search of the same shape (cphb_search_knn / cphb_search_radius of its query rows against the cloud) and the client's own
kernels -- nothing more.  Fused EstimateNormals launches the index build and its one kernel; its block form also orders
its queries as the search does."""
import ctypes as C

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

from cupoch_b200 import _lib
from cupoch_b200.testing import datagen
from cupoch_b200.utility import DeviceArray

N = 20_000
FIRST, COUNT = 5_000, 10_000  # block of the range form of EstimateNormals


@pytest.fixture(scope="module")
def cloud():
    pts, nrm = datagen.surface(N, 12)
    return (DeviceArray.from_numpy(pts), DeviceArray.from_numpy(nrm),
            DeviceArray.from_numpy(datagen.texture(pts, 5)))


def launches(fn):
    """launches of one call of fn, after one warm-up call"""
    L = _lib.lib()
    fn()
    _lib.check(L.cphb_stream_synchronize(None))
    before = L.cphb_launch_count()
    fn()
    _lib.check(L.cphb_stream_synchronize(None))
    return L.cphb_launch_count() - before


@pytest.fixture(scope="module")
def base(cloud):
    """launches of the index build, and of a standalone search (knn, radius, max_nn) of `nq` query rows"""
    L = _lib.lib()
    pts = cloud[0]

    def build():
        h = C.c_void_p()
        _lib.check(L.cphb_index_create(pts.ptr, N, None, C.byref(h)))
        _lib.check(L.cphb_stream_synchronize(None))
        L.cphb_index_destroy(h)

    def search(knn, radius, max_nn, nq=N, first=0):
        k = knn if knn > 0 else max_nn
        h = C.c_void_p()
        _lib.check(L.cphb_index_create(pts.ptr, N, None, C.byref(h)))
        idx, d2 = DeviceArray((nq, k), np.int32), DeviceArray((nq, k), np.float32)
        q = pts.ptr + 12 * first
        if knn > 0:
            n = launches(lambda: _lib.check(L.cphb_search_knn(h, q, nq, knn, idx.ptr, d2.ptr, None, None)))
        else:
            n = launches(lambda: _lib.check(L.cphb_search_radius(h, q, nq, radius, max_nn, idx.ptr, d2.ptr, None, None)))
        L.cphb_index_destroy(h)
        return n

    n_build = launches(build)
    assert n_build > 0
    return n_build, search


@pytest.mark.parametrize("knn,radius,max_nn", [(30, 0.0, 0), (0, 0.02, 30)])
def test_fpfh(cloud, base, knn, radius, max_nn):
    pts, nrm, _ = cloud
    out = DeviceArray((N, 33), np.float32)
    L = _lib.lib()
    got = launches(lambda: _lib.check(L.cphb_compute_fpfh_feature(pts.ptr, nrm.ptr, N, knn, radius, max_nn, out.ptr, None)))
    build, search = base
    assert got == build + search(knn, radius, max_nn) + 2


def test_color_gradient(cloud, base):
    pts, nrm, col = cloud
    out = DeviceArray((N, 3), np.float32)
    L = _lib.lib()
    got = launches(lambda: _lib.check(L.cphb_color_gradient(pts.ptr, nrm.ptr, col.ptr, N, 0.02, 30, out.ptr, None)))
    build, search = base
    assert got == build + search(0, 0.02, 30) + 1


def test_gaussian_filter(cloud, base):
    pts, nrm, col = cloud
    o = [DeviceArray((N, 3), np.float32) for _ in range(3)]
    m = C.c_size_t(0)
    L = _lib.lib()
    got = launches(lambda: _lib.check(L.cphb_gaussian_filter(pts.ptr, nrm.ptr, col.ptr, N, 0.02, 1e-4, 30, o[0].ptr, o[1].ptr,
                                                             o[2].ptr, C.byref(m), None)))
    build, search = base
    assert m.value == N
    assert got == build + search(0, 0.02, 30) + 1


def test_radius_outliers(cloud, base):
    pts = cloud[0]
    out, m = DeviceArray((N,), np.int32), C.c_size_t(0)
    L = _lib.lib()
    got = launches(lambda: _lib.check(L.cphb_remove_radius_outliers(pts.ptr, N, 8, 0.02, out.ptr, C.byref(m), None)))
    build, search = base
    assert 0 < m.value <= N
    assert got == build + search(0, 0.02, 9) + 1 + 3  # + the compaction


def test_statistical_outliers(cloud, base):
    pts = cloud[0]
    out, m, stats = DeviceArray((N,), np.int32), C.c_size_t(0), (C.c_float * 3)()
    L = _lib.lib()
    got = launches(lambda: _lib.check(L.cphb_remove_statistical_outliers(pts.ptr, N, 20, 2.0, out.ptr, C.byref(m), stats,
                                                                         None)))
    build, search = base
    assert 0 < m.value <= N
    assert got == build + search(20, 0.0, 0) + 6 + 3  # + the compaction


def test_dbscan(cloud, base):
    pts = cloud[0]
    labels, ncl = DeviceArray((N,), np.int32), C.c_int(0)
    L = _lib.lib()
    got = launches(lambda: _lib.check(L.cphb_cluster_dbscan(pts.ptr, N, 0.02, 10, 100, labels.ptr, C.byref(ncl), None)))
    build, search = base
    assert got == build + search(0, 0.02, 101) + 2


@pytest.mark.parametrize("knn,radius,max_nn", [(30, 0.0, 0), (0, 0.02, 30)])
def test_estimate_normals(cloud, base, monkeypatch, knn, radius, max_nn):
    pts = cloud[0]
    out = DeviceArray((N, 3), np.float32)
    L = _lib.lib()

    def whole():
        _lib.check(L.cphb_estimate_normals(pts.ptr, N, knn, radius, max_nn, out.ptr, None))

    def block():
        _lib.check(L.cphb_estimate_normals_range(pts.ptr, N, knn, radius, max_nn, FIRST, COUNT, out.ptr, None))

    build, search = base
    assert launches(whole) == build + 1  # fused: queries in index order, no ordering pass, no table
    assert launches(block) == build + search(knn, radius, max_nn, COUNT, FIRST)  # ordering pass + the fused kernel
    monkeypatch.setenv("CPHB_NORMALS_UNFUSED", "1")  # two-pass: table, then normals_kernel
    assert launches(whole) == build + search(knn, radius, max_nn) + 1
    assert launches(block) == build + search(knn, radius, max_nn, COUNT, FIRST) + 1
