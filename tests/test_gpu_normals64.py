"""GPU: EstimateNormals on the device -- the fused kernel, the two-pass form (CPHB_NORMALS_UNFUSED=1) and the block form
cphb_estimate_normals_range -- on the inputs of tests/test_oracle_normals64.py and at 1 M points.  On every cloud all
three equal the CPU oracle bit for bit and satisfy the float64 PCA of cupoch_b200/testing/normals64.py over the
device's own neighbour lists (KDTreeFlann, itself pinned to the oracle and to FLANN).  The device GICP covariances
equal the oracle's on the normals of the analytic check."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing import datagen
from cupoch_b200.testing import normals64 as N
from cupoch_b200.utility import DeviceArray

G = cph.geometry
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsdf_rgbd_known.npz")


def _normals(orc, monkeypatch, p, knn=0, radius=0.0, max_nn=0, label=""):
    """device normals (fused, two-pass, and the block [n / 3, n - n / 5)) == oracle, and within normals64's bounds"""
    n = len(p)
    param = G.KDTreeSearchParamKNN(knn) if knn > 0 else G.KDTreeSearchParamRadius(radius, max_nn)
    pc = G.PointCloud(p)
    pc.estimate_normals(param)
    fused = pc.normals.cpu()
    monkeypatch.setenv("CPHB_NORMALS_UNFUSED", "1")
    pc.estimate_normals(param)
    two = pc.normals.cpu()
    monkeypatch.delenv("CPHB_NORMALS_UNFUSED")
    o = orc.estimate_normals(p, knn=knn, radius=radius, max_nn=max_nn)
    np.testing.assert_array_equal(fused, o)
    np.testing.assert_array_equal(two, o)
    lo, hi = n // 3, n - n // 5
    if hi > lo:
        out = DeviceArray((hi - lo, 3), np.float32)
        _lib.check(_lib.lib().cphb_estimate_normals_range(pc.points.ptr, n, knn, radius, max_nn, lo, hi - lo, out.ptr, None))
        np.testing.assert_array_equal(out.cpu(), o[lo:hi])
    tree = G.KDTreeFlann(pc)
    _, idx, _ = tree.search_knn(pc.points, knn) if knn > 0 else tree.search_radius(pc.points, radius, max_nn)
    idx = idx.cpu()
    return fused, idx, N.check_normals(fused, p, idx, label)


@pytest.mark.parametrize("offset", [0.0, 1.0, 10.0, 100.0, 1000.0])
def test_offset(orc, monkeypatch, offset):
    p, _ = datagen.surface(100_000, 5)
    q = (p.astype(np.float64) + offset).astype(np.float32)
    _normals(orc, monkeypatch, q, knn=20, label="offset %g knn" % offset)
    _normals(orc, monkeypatch, q, radius=0.01, max_nn=30, label="offset %g radius" % offset)


@pytest.mark.parametrize("scale", [1e-5, 10.0])
def test_scale(orc, monkeypatch, scale):
    p, _ = datagen.surface(20_000, 6)
    _normals(orc, monkeypatch, (p * np.float32(scale)).astype(np.float32), knn=30, label="scale %g" % scale)


PLANES = [("x", 0.01, 0.5), ("y", 0.01, 0.5), ("z", 0.01, 0.5), ("xy", 0.01, 0.5), ("random", 0.01, 0.5),
          ("x", 10.0, 5.0)]


@pytest.mark.parametrize("plane,spacing,c", PLANES, ids=["%s-%g" % (a, b) for a, b, _ in PLANES])
def test_lattice_plane(orc, monkeypatch, plane, spacing, c):
    p, nrm = N.lattice_plane(plane, spacing=spacing, c=c)
    n, _, _ = _normals(orc, monkeypatch, p, knn=20, label="plane %s knn" % plane)
    assert (np.abs(n.astype(np.float64) @ nrm) > 1 - 1e-5).all()
    _normals(orc, monkeypatch, p, radius=2.5 * spacing, max_nn=30, label="plane %s radius" % plane)
    n, _, _ = _normals(orc, monkeypatch, N.duplicated(p), knn=20, label="plane %s duplicated" % plane)
    assert (np.abs(n.astype(np.float64) @ nrm) > 1 - 1e-5).all()


@pytest.mark.parametrize("direction", [(0, 0, 1), (0.3, -0.5, 0.8)], ids=["axis", "random"])
def test_line(orc, monkeypatch, direction):
    p = N.line(500, direction)
    d = np.asarray(direction, np.float64) / np.linalg.norm(direction)
    for knn in (5, 30):
        n, _, info = _normals(orc, monkeypatch, p, knn=knn, label="line %s k%d" % (direction, knn))
        assert info["line_checked"] == len(p) and (np.abs(n.astype(np.float64) @ d) < 1e-5).all()


def test_isotropic_cube_and_duplicates(orc, monkeypatch):
    p = N.cube_lattice(12)
    for knn in (7, 27):
        _, _, info = _normals(orc, monkeypatch, p, knn=knn, label="cube k%d" % knn)
        assert info["free"] >= 1000
    _normals(orc, monkeypatch, p, radius=0.13, max_nn=30, label="cube radius")
    p = N.duplicated(datagen.surface(20_000, 7)[0])
    _, _, info = _normals(orc, monkeypatch, p, knn=3, label="duplicates k3")
    assert info["zero"] == len(p)
    _normals(orc, monkeypatch, p, knn=20, label="duplicates k20")
    _normals(orc, monkeypatch, p, radius=0.015, max_nn=256, label="duplicates radius")


def test_depth_frames(orc, monkeypatch):
    """the reference's five real depth frames through create_from_depth_image (the device's own projection)"""
    z = np.load(GOLDEN)
    K = cph.camera.PinholeCameraIntrinsic(cph.camera.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    for i in range(5):
        pd = G.PointCloud.create_from_depth_image(G.Image(z["depth"][i]), K, z["extrinsics"][i], 1000.0, 4.0, 1)
        p = pd.points.cpu()
        assert len(p) > 200_000
        _normals(orc, monkeypatch, p, knn=30, label="frame %d knn" % i)
        _normals(orc, monkeypatch, p, radius=0.01, max_nn=30, label="frame %d radius" % i)


@pytest.mark.parametrize("knn", [2, 3, 5, 30, 100])
def test_knn_shapes(orc, monkeypatch, knn):
    p, _ = datagen.surface(100_000, 8)
    _normals(orc, monkeypatch, (p.astype(np.float64) + 10.0).astype(np.float32), knn=knn, label="knn %d" % knn)


@pytest.mark.parametrize("radius,max_nn", [(0.007, 3), (0.007, 30), (0.02, 30), (0.02, 256), (0.05, 256)])
def test_radius_shapes(orc, monkeypatch, radius, max_nn):
    """max_nn 3, 30 and 256 (the limit); (0.02, 30) and (0.05, 256) truncate most lists, (0.007, 30) few"""
    p, _ = datagen.surface(100_000, 9)
    p = (p.astype(np.float64) + 10.0).astype(np.float32)
    _, idx, _ = _normals(orc, monkeypatch, p, radius=radius, max_nn=max_nn, label="radius %g max_nn %d" % (radius, max_nn))
    full = (idx >= 0).all(1).mean()
    if (radius, max_nn) in ((0.02, 30), (0.05, 256)):
        assert full > 0.9
    if (radius, max_nn) == (0.007, 30):
        assert full < 0.5


@pytest.mark.parametrize("size", [1, 2, 3, 31, 32, 33, 1025, 100_000, 1_000_000])
def test_sizes(orc, monkeypatch, size):
    p, _ = datagen.surface(size, size, extent=max(1.0, np.sqrt(size / 1e5)))
    _normals(orc, monkeypatch, p, knn=30, label="n=%d knn" % size)
    _normals(orc, monkeypatch, p, radius=0.01, max_nn=30, label="n=%d radius" % size)


def test_no_neighbours(orc):
    """knn 0 and max_nn 0: every normal (0, 0, 1), as the oracle"""
    p, _ = datagen.surface(1_000, 10)
    pc = G.PointCloud(p)
    for param in (G.KDTreeSearchParamKNN(0), G.KDTreeSearchParamRadius(0.1, 0)):
        pc.estimate_normals(param)
        np.testing.assert_array_equal(pc.normals.cpu(), np.tile(np.float32([0, 0, 1]), (len(p), 1)))
    np.testing.assert_array_equal(pc.normals.cpu(), orc.estimate_normals(p, knn=0, radius=0.1, max_nn=0))


def test_gicp_covariances(orc):
    """the device's covariances_from_normals equals the oracle's on the 200 k normals of the CPU file's analytic check"""
    nrm = datagen.unit_normals(200_000, 11)
    nrm[:6] = [[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, 0, -1], [-0.99, np.sqrt(1 - 0.99 ** 2), 0], [-0.98, 0.199, 0]]
    pc = G.PointCloud(datagen.uniform_cube(len(nrm), 1))
    pc.normals = nrm
    cov = cph.registration._with_covariances(pc, 1e-3).covariances.cpu()
    np.testing.assert_array_equal(cov, orc.covariances_from_normals(nrm, 1e-3))
    A, branch = N.gicp_cov64(nrm, 1e-3)
    assert (np.abs(cov[~branch] - A[~branch]).max((1, 2)) * (1.0 + nrm[~branch, 0]) <= 2.0 ** -18).all()
