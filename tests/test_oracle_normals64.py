"""CPU: the oracle's EstimateNormals against the float64 PCA of cupoch_b200/testing/normals64.py over the oracle's own
neighbour lists -- far from the origin, at tiny and large scales, on axis-aligned, diagonal and rotated lattice planes,
on lines, isotropic and duplicated lattices, the real depth frames, every search shape and sizes across warp and leaf
edges -- and the GICP covariances of covariances_from_normals against the analytic I - (1 - eps) n n^T."""
import os

import numpy as np
import pytest

from cupoch_b200.testing import datagen
from cupoch_b200.testing import normals64 as N

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsdf_rgbd_known.npz")
PRIMESENSE = np.array([[525.0, 0.0, 319.5], [0.0, 525.0, 239.5], [0.0, 0.0, 1.0]])


def _normals(orc, p, knn=0, radius=0.0, max_nn=0, label=""):
    """the oracle's normals, equal to its normals over the lists its own search returns, checked against normals64"""
    k = knn if knn > 0 else max_nn
    idx = orc.search(p, p, k, radius if knn == 0 else -1.0, kdtree=True)[0]
    n = orc.estimate_normals(p, knn=knn, radius=radius, max_nn=max_nn)
    np.testing.assert_array_equal(n, orc.normals_from_neighbors(p, idx))
    return n, idx, N.check_normals(n, p, idx, label)


@pytest.mark.parametrize("offset", [0.0, 1.0, 10.0, 100.0, 1000.0])
def test_offset(orc, offset):
    """a 1 m surface shifted by `offset` along every axis: the covariance's E[xx^T] - E[x]E[x]^T cancels |m|^2"""
    p, _ = datagen.surface(20_000, 5)
    q = (p.astype(np.float64) + offset).astype(np.float32)
    _normals(orc, q, knn=20, label="offset %g knn" % offset)
    _normals(orc, q, radius=0.03, max_nn=30, label="offset %g radius" % offset)


@pytest.mark.parametrize("scale", [1e-5, 10.0])
def test_scale(orc, scale):
    p, _ = datagen.surface(20_000, 6)
    _normals(orc, (p * np.float32(scale)).astype(np.float32), knn=30, label="scale %g" % scale)


PLANES = [("x", 0.01, 0.5), ("y", 0.01, 0.5), ("z", 0.01, 0.5), ("xy", 0.01, 0.5), ("random", 0.01, 0.5),
          ("x", 10.0, 5.0)]


@pytest.mark.parametrize("plane,spacing,c", PLANES, ids=["%s-%g" % (a, b) for a, b, _ in PLANES])
def test_lattice_plane(orc, plane, spacing, c):
    """axis-aligned lattice planes: FastEigen3x3's second eigenvector divides 0 by 0 (signf of an exactly zero
    projection) and the normal must not become (0, 0, 1)"""
    p, nrm = N.lattice_plane(plane, spacing=spacing, c=c)
    n, _, _ = _normals(orc, p, knn=20, label="plane %s knn" % plane)
    assert (np.abs(n.astype(np.float64) @ nrm) > 1 - 1e-5).all()
    _normals(orc, p, radius=2.5 * spacing, max_nn=30, label="plane %s radius" % plane)


def test_lattice_plane_duplicated(orc):
    p, nrm = N.lattice_plane("x")
    n, _, _ = _normals(orc, N.duplicated(p), knn=20, label="plane x duplicated")
    assert (np.abs(n.astype(np.float64) @ nrm) > 1 - 1e-5).all()


@pytest.mark.parametrize("direction", [(0, 0, 1), (0.3, -0.5, 0.8)], ids=["axis", "random"])
@pytest.mark.parametrize("knn", [5, 30])
def test_line(orc, direction, knn):
    """lam0 == lam1: any normal perpendicular to the line is right"""
    p = N.line(500, direction)
    n, _, info = _normals(orc, p, knn=knn, label="line %s k%d" % (direction, knn))
    assert info["line_checked"] == len(p)
    d = np.asarray(direction, np.float64) / np.linalg.norm(direction)
    assert (np.abs(n.astype(np.float64) @ d) < 1e-5).all()


@pytest.mark.parametrize("knn", [7, 27])
def test_isotropic_cube(orc, knn):
    """inner points of a cube lattice: their 7 or 27 nearest have an isotropic covariance (only finite and unit)"""
    p = N.cube_lattice(12)
    _, _, info = _normals(orc, p, knn=knn, label="cube k%d" % knn)
    assert info["free"] >= 1000
    _normals(orc, p, radius=0.13, max_nn=30, label="cube radius")


def test_duplicates(orc):
    """every point 4 times: at k = 3 each list is three copies of one point (zero covariance, (1, 0, 0)); at k = 20 five
    distinct points with repeats"""
    p = N.duplicated(datagen.surface(5_000, 7)[0])
    _, _, info = _normals(orc, p, knn=3, label="duplicates k3")
    assert info["zero"] == len(p)
    _normals(orc, p, knn=20, label="duplicates k20")
    _normals(orc, p, radius=0.03, max_nn=256, label="duplicates radius")


@pytest.mark.parametrize("frame", range(5))
def test_depth_frames(frame):
    """the reference's real depth frames through CreateFromDepthImage, in world coordinates (metres from the origin)"""
    from oracle import depth_cloud_py as D
    from oracle import oracle_py as orc
    z = np.load(GOLDEN)
    p, _, _ = D.depth_to_points(z["depth"][frame], PRIMESENSE, z["extrinsics"][frame], 1000.0, 4.0, 2)
    assert len(p) > 50_000
    _normals(orc, p, knn=30, label="frame %d knn" % frame)
    _normals(orc, p, radius=0.02, max_nn=30, label="frame %d radius" % frame)


@pytest.mark.parametrize("knn", [2, 3, 5, 30, 100])
def test_knn_shapes(orc, knn):
    p, _ = datagen.surface(20_000, 8)
    _normals(orc, (p.astype(np.float64) + 10.0).astype(np.float32), knn=knn, label="knn %d" % knn)


@pytest.mark.parametrize("radius,max_nn", [(0.02, 3), (0.02, 30), (0.05, 30), (0.05, 256), (0.1, 256)])
def test_radius_shapes(orc, radius, max_nn):
    """max_nn 3, 30 and 256 (the limit); (0.05, 30) and (0.1, 256) truncate most lists, the others few"""
    p, _ = datagen.surface(20_000, 9)
    p = (p.astype(np.float64) + 10.0).astype(np.float32)
    _, idx, _ = _normals(orc, p, radius=radius, max_nn=max_nn, label="radius %g max_nn %d" % (radius, max_nn))
    full = (idx >= 0).all(1).mean()
    if (radius, max_nn) in ((0.05, 30), (0.1, 256)):
        assert full > 0.9
    if max_nn == 30 and radius == 0.02:
        assert full < 0.5


@pytest.mark.parametrize("size", [1, 2, 3, 31, 32, 33, 1025, 100_000, 1_000_000])
def test_sizes(orc, size):
    p, _ = datagen.surface(size, size, extent=max(1.0, np.sqrt(size / 1e5)))
    _normals(orc, p, knn=30, label="n=%d knn" % size)
    if size <= 100_000:
        _normals(orc, p, radius=0.05, max_nn=30, label="n=%d radius" % size)


def test_no_neighbours(orc):
    """k = 0 (knn 0 and max_nn 0) and radius lists with fewer than 3 points: (0, 0, 1)"""
    p, _ = datagen.surface(1_000, 10)
    n = orc.estimate_normals(p, knn=0, radius=0.1, max_nn=0)
    N.check_normals(n, p, np.zeros((len(p), 0), np.int32), "k = 0")
    _, _, info = _normals(orc, p, radius=1e-4, max_nn=30, label="tiny radius")
    assert info["few"] == len(p)


def test_gicp_covariances(orc):
    """covariances_from_normals against I - (1 - eps) n n^T.  Outside the reference's n_x < -0.99 branch the error of
    its Rodrigues form is the few 2^-24 by which a float32 unit normal's squared length misses 1, and a few roundings,
    divided by 1 + n_x (at least 0.01): within 2^-18 / (1 + n_x).
    Inside it the reference returns diag(eps, 1, 1) for every normal (mirrored, DESIGN.md section 4)."""
    eps = 1e-3
    nrm = datagen.unit_normals(200_000, 11)
    nrm[:6] = [[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, 0, -1], [-0.99, np.sqrt(1 - 0.99 ** 2), 0], [-0.98, 0.199, 0]]
    cov = orc.covariances_from_normals(nrm, eps).astype(np.float64)
    A, branch = N.gicp_cov64(nrm, eps)
    out = ~branch
    err = np.abs(cov - A).max((1, 2))
    scaled = err[out] * (1.0 + nrm[out, 0].astype(np.float64))
    print("gicp covariances: %d in the branch, max error outside %.3g, max error (1 + n_x) / 2^-18 %.3g"
          % (int(branch.sum()), float(err[out].max()), float(scaled.max() / 2.0 ** -18)))
    assert (scaled <= 2.0 ** -18).all()
    assert 500 < branch.sum() < 2000
    np.testing.assert_array_equal(cov[branch], np.broadcast_to(np.diag(np.float32([eps, 1, 1])), (int(branch.sum()), 3, 3)))
    assert err[branch].max() > 0.1  # what the branch costs: up to 0.139 from the analytic covariance
