"""GPU: PointCloud::FarthestPointDownSample (csrc/fps.cu).

- The pick sequence and the final running distances equal the CPU oracle bit for bit: at sizes around warp and block
  boundaries, on both sides of the shared-memory residency switch (SMs * 14336 points) and at 10 M points, and for
  every sample count from 1 to n on small clouds.
- The final distances equal, bit for bit, the nearest-neighbour d2 that KDTreeFlann over the picked points returns
  (both use dist2, and dist2 does not depend on which point is subtracted from which).
- Integer lattices equal an int64 loop with np.argmax (the tie rule), the quirks hold through the Python method,
  attributes are gathered row for row, calls repeat bit for bit, and the whole loop is one launch."""
import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing import datagen
from cupoch_b200.utility import DeviceArray
from test_oracle_fps import int64_fps, lattice

SMEM_POINTS = 14336  # fps.cu FPS_SMEM_POINTS: resident points per block, one block per SM


@pytest.fixture(scope="module")
def fpso():
    """the FarthestPointDownSample restatement (oracle/fps.c)"""
    from oracle import fps_py
    fps_py.build()
    return fps_py


def device_fps(pc, k):
    """the ABI call on a PointCloud -> (indices [k], final running distances [n])"""
    n = len(pc)
    idx, d2 = DeviceArray((k,), np.int32), DeviceArray((n,), np.float32)
    _lib.check(_lib.lib().cphb_farthest_point_down_sample(pc.points.ptr, n, k, idx.ptr, d2.ptr, None))
    return idx.cpu(), d2.cpu()


def check_oracle(fpso, pts, k):
    idx, d2 = device_fps(cph.geometry.PointCloud(pts), k)
    o_idx, o_d2 = fpso.farthest_point_down_sample(pts, k)
    np.testing.assert_array_equal(idx, o_idx)
    np.testing.assert_array_equal(d2.view(np.uint32), o_d2.view(np.uint32))
    return idx, d2


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1023, 1024, 1025, 100_000, 1_000_000])
def test_equals_oracle(fpso, n):
    pts = datagen.surface(n, 40 + n % 97)[0]
    k = min(n, 1024) if n < 1_000_000 else 256
    check_oracle(fpso, pts, k)


@pytest.mark.parametrize("n", [1, 2, 31, 33, 100])
def test_every_sample_count(fpso, n):
    pts = datagen.uniform_cube(n, 3, lo=(-1, -1, -1))
    for k in range(1, n + 4):
        check_oracle(fpso, pts, k)


def test_residency_switch(fpso):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    edge = sms * SMEM_POINTS
    pts = datagen.uniform_cube(edge + 1, 12, hi=(3, 2, 1))
    for n in (edge - 1, edge, edge + 1):
        check_oracle(fpso, pts[:n], 96)


def test_10m(fpso):
    pts = datagen.uniform_cube(10_000_000, 13, hi=(4, 4, 1))
    check_oracle(fpso, pts, 256)


@pytest.mark.parametrize("n,k", [(5000, 300), (300_000, 2000), (2_500_000, 200)])
def test_d2_equals_nearest_neighbour_search(n, k):
    pts = datagen.surface(n, 21)[0]
    pc = cph.geometry.PointCloud(pts)
    idx, d2 = device_fps(pc, k)
    tree = cph.geometry.KDTreeFlann(cph.geometry.PointCloud(pts[idx]))
    _, _, nn_d2 = tree.search_knn(pc.points, 1)
    np.testing.assert_array_equal(d2.view(np.uint32), nn_d2.cpu().reshape(-1).view(np.uint32))


@pytest.mark.parametrize("n,k,seed", [(500, 505, 2), (20000, 600, 4), (200_000, 300, 5)])
def test_lattice_equals_int64_loop(n, k, seed):
    P = lattice(n, seed)
    idx, d2 = device_fps(cph.geometry.PointCloud(P.astype(np.float32)), k)
    ref_idx, ref_dist = int64_fps(P, k)
    np.testing.assert_array_equal(idx, ref_idx)
    np.testing.assert_array_equal(d2.astype(np.int64), ref_dist)


def test_python_sample_counts(fpso, capsys):
    pts = datagen.surface(3000, 7)[0]
    pc = cph.geometry.PointCloud(pts)
    assert len(pc.farthest_point_down_sample(0)) == 0
    np.testing.assert_array_equal(pc.farthest_point_down_sample(1).points.cpu(), pts[:1])
    full = pc.farthest_point_down_sample(len(pts))  # the whole cloud, in its original order
    np.testing.assert_array_equal(full.points.cpu(), pts)
    assert full.points.ptr != pc.points.ptr
    capsys.readouterr()
    more = pc.farthest_point_down_sample(len(pts) + 5)
    assert "Illegal number of samples" in capsys.readouterr().err
    o_idx, _ = fpso.farthest_point_down_sample(pts, len(pts) + 5)
    np.testing.assert_array_equal(more.points.cpu(), pts[o_idx])
    assert o_idx[-5:].tolist() == [0] * 5


def test_python_degenerate_clouds(capsys):
    empty = cph.geometry.PointCloud()
    assert len(empty.farthest_point_down_sample(0)) == 0
    assert len(empty.farthest_point_down_sample(3)) == 0
    assert "Illegal number of samples" in capsys.readouterr().err
    one = cph.geometry.PointCloud(np.array([[1, 2, 3]], np.float32))
    np.testing.assert_array_equal(one.farthest_point_down_sample(3).points.cpu(), np.tile([[1, 2, 3]], (3, 1)))
    same = cph.geometry.PointCloud(np.full((5000, 3), 0.5, np.float32))
    assert len(same.farthest_point_down_sample(7)) == 7
    with pytest.raises(ValueError):
        one.farthest_point_down_sample(-1)


@pytest.mark.parametrize("bad", [[np.nan, 0, 0], [0, np.inf, 0]])
def test_python_non_finite_point_repeats(fpso, bad):
    pts = datagen.uniform_cube(5000, 9)
    pts[37] = bad
    pc = cph.geometry.PointCloud(pts)
    idx, d2 = device_fps(pc, 8)
    assert idx.tolist() == [0] + [37] * 7
    o_idx, o_d2 = fpso.farthest_point_down_sample(pts, 8)
    np.testing.assert_array_equal(d2.view(np.uint32), o_d2.view(np.uint32))
    out = pc.farthest_point_down_sample(8).points.cpu()
    np.testing.assert_array_equal(out, pts[o_idx])


def test_attributes_gathered_row_for_row(fpso):
    pts, nrm = datagen.surface(20000, 31)
    col = datagen.texture(pts, 3)
    pc = cph.geometry.PointCloud(pts)
    pc.normals, pc.colors = nrm, col
    pc.covariances = np.tile(np.eye(3, dtype=np.float32), (len(pts), 1, 1))
    out = pc.farthest_point_down_sample(500)
    o_idx, _ = fpso.farthest_point_down_sample(pts, 500)
    np.testing.assert_array_equal(out.points.cpu(), pts[o_idx])
    np.testing.assert_array_equal(out.normals.cpu(), nrm[o_idx])
    np.testing.assert_array_equal(out.colors.cpu(), col[o_idx])
    assert not out.has_covariances()  # SelectByIndex gathers points, normals and colours only
    full = pc.farthest_point_down_sample(len(pts))  # == n: the reference's copy, covariances included
    np.testing.assert_array_equal(full.normals.cpu(), nrm)
    np.testing.assert_array_equal(full.colors.cpu(), col)
    assert full.has_covariances()


def test_repeatable():
    pc = cph.geometry.PointCloud(datagen.surface(1_000_000, 8)[0])
    a, b = device_fps(pc, 2048), device_fps(pc, 2048)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_one_launch_whatever_the_sample_count():
    L = _lib.lib()
    for n in (50_000, 5_000_000):
        pc = cph.geometry.PointCloud(datagen.uniform_cube(n, 4))
        device_fps(pc, 2)  # warm-up
        grown = []
        for k in (10, 1000):
            before = L.cphb_launch_count()
            device_fps(pc, k)
            grown.append(L.cphb_launch_count() - before)
        assert grown[0] == grown[1] == 1
