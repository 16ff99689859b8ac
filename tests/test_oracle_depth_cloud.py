"""CPU: the CreateFromDepthImage / CreateFromRGBDImage restatement (oracle/depth_cloud.c) against float64 restatements
and analytic scenes.

- Fronto-parallel and tilted planes and a sphere rendered to depth: every point lies on the surface; points agree with a
  float64 back-projection; structured normals of a plane equal its normal, turned to z <= 0, and are 0 on the border.
- The uint16 conversion rule is cphb_rgbd_convert's (oracle/tsdf.c's depth_to_float); stride sampling at odd sizes,
  depth_cutoff, the colour rules, NaN rows when project_valid_depth_only is off, and the float64 pose.
"""
import numpy as np
import pytest

from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import depth_cloud_py as D
from oracle import tsdf_py as T


def K_of(w, h, f=None):
    f = f or 0.9 * w
    return np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], np.float32)


def rigid(seed, t_scale=0.5):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    R = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                  [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                  [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])
    E = np.eye(4, dtype=np.float32)
    E[:3, :3] = R
    E[:3, 3] = rng.normal(size=3) * t_scale
    return E


def back_project64(depth_m, K, E, stride=1):
    """float64: every sampled pixel's world point, and the mask of d > 0"""
    h, w = depth_m.shape
    sh, sw = h // stride, w // stride
    rows, cols = np.meshgrid(np.arange(sh) * stride, np.arange(sw) * stride, indexing="ij")
    z = depth_m[rows, cols].astype(np.float64)
    K = np.asarray(K, np.float64)
    x = (cols - K[0, 2]) * z / K[0, 0]
    y = (rows - K[1, 2]) * z / K[1, 1]
    P = np.linalg.inv(np.asarray(E, np.float64))
    cam = np.stack([x, y, z, np.ones_like(z)], -1).reshape(-1, 4)
    return (cam @ P.T)[:, :3], (z > 0).reshape(-1)


def test_pose_is_the_float64_inverse():
    for seed in range(20):
        E = rigid(seed)
        if seed % 2:
            E[:3, :3] *= np.float32(1.0 + 0.3 * seed)  # a non-rigid extrinsic
            E[0, 1] += np.float32(0.2)
        P = D.pose(E)
        ref = np.linalg.inv(E.astype(np.float64))[:3].astype(np.float32)
        np.testing.assert_array_equal(P, ref)
    S = np.eye(4, dtype=np.float32)
    S[2, 2] = 0
    assert D.pose(S) is None
    with pytest.raises(ValueError):
        D.depth_to_points(np.ones((4, 4), np.float32), K_of(4, 4), S)


def test_fronto_parallel_plane():
    w, h, Z = 37, 29, np.float32(1.7)
    K = K_of(w, h)
    depth = np.full((h, w), Z, np.float32)
    p, n, _ = D.depth_to_points(depth, K, compute_normals=True)
    assert len(p) == w * h
    assert np.all(p[:, 2] == Z)
    ref, _ = back_project64(depth, K, np.eye(4))
    assert np.max(np.abs(p - ref)) <= 2e-6 * Z
    n = n.reshape(h, w, 3)
    np.testing.assert_array_equal(n[1:-1, 1:-1].reshape(-1, 3), np.tile(np.float32([0, 0, -1]), ((h - 2) * (w - 2), 1)))
    for border in (n[0], n[-1], n[:, 0], n[:, -1]):
        assert not border.any()


def plane_depth(K, w, h, nrm, off):
    """camera-frame depth of the plane n . X = off, seen through K"""
    Ki = np.linalg.inv(np.asarray(K, np.float64))
    uu, vv = np.meshgrid(np.arange(w), np.arange(h))
    rays = np.stack([uu, vv, np.ones_like(uu)], -1) @ Ki.T
    return (off / (rays @ nrm)).astype(np.float32)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_tilted_plane_points_and_normals(seed):
    w, h = 41, 31
    K = K_of(w, h)
    rng = np.random.default_rng(seed)
    nc = np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4), -1.0])
    nc /= np.linalg.norm(nc)
    off = -2.0  # n . X = -2: a plane in front of the camera, its normal towards the camera
    depth = plane_depth(K, w, h, nc, off)
    assert np.all(depth > 0)
    E = rigid(10 + seed)
    p, n, _ = D.depth_to_points(depth, K, E, compute_normals=True)
    P = np.linalg.inv(E.astype(np.float64))
    nw = P[:3, :3] @ nc  # the plane in the world: nw . X = off + nw . t
    dw = off + nw @ P[:3, 3]
    assert np.max(np.abs(p.astype(np.float64) @ nw - dw)) < 5e-6 * 4
    ref, _ = back_project64(depth, K, E)
    assert np.max(np.abs(p - ref)) < 2e-5
    inner = n.reshape(h, w, 3)[1:-1, 1:-1].reshape(-1, 3).astype(np.float64)
    want = nw if nw[2] <= 0 else -nw
    assert np.max(np.abs(inner - want)) < 2e-3
    assert np.all(inner[:, 2] <= 0)


def test_sphere_points_lie_on_the_sphere_and_skip_misses():
    w, h, R = 64, 48, 0.6
    for K, E in ring_cameras(3, w, h):
        depth = sphere_depth(K, E, w, h, R)
        p, n, _ = D.depth_to_points(depth, K, E, compute_normals=True)
        assert len(p) == np.count_nonzero(depth > 0) > 100
        assert np.max(np.abs(np.linalg.norm(p.astype(np.float64), axis=1) - R)) < 2e-5
        ref, keep = back_project64(depth, K, E)
        assert np.max(np.abs(p - ref[keep])) < 2e-5
        # normals on the visible side point back towards the camera's side of the sphere where they are not zero
        live = np.any(n != 0, 1)
        assert np.all(n[live, 2] <= 0)


def test_uint16_uses_the_rgbd_conversion_rule():
    w, h = 23, 17
    rng = np.random.default_rng(5)
    raw = rng.integers(0, 5000, (h, w), dtype=np.uint16)
    raw[0, :5] = 0
    for scale, trunc in ((1000.0, 3.0), (5000.0, 4.0), (999.9, 2.5)):
        ref = T.depth_to_float(raw, scale, trunc)
        p, _, _ = D.depth_to_points(raw, K_of(w, h), depth_scale=scale, depth_trunc=trunc, project_valid_depth_only=False)
        got = p[:, 2].reshape(h, w)
        keep = ref > 0
        np.testing.assert_array_equal(got[keep], ref[keep])
        assert np.all(np.isnan(got[~keep]))
        q, _, _ = D.depth_to_points(ref, K_of(w, h))
        np.testing.assert_array_equal(q, p[keep.reshape(-1)])


@pytest.mark.parametrize("stride", [1, 3, 4])
def test_stride_samples_every_stride_th_pixel(stride):
    w, h = 47, 35
    rng = np.random.default_rng(stride)
    depth = rng.uniform(0.5, 3.0, (h, w)).astype(np.float32)
    depth[rng.random((h, w)) < 0.2] = 0
    E = rigid(stride)
    K = K_of(w, h)
    p, _, _ = D.depth_to_points(depth, K, E, stride=stride)
    ref, keep = back_project64(depth, K, E, stride)
    assert len(p) == np.count_nonzero(keep)
    assert np.max(np.abs(p - ref[keep])) < 2e-5
    full, _, _ = D.depth_to_points(depth, K, E, stride=stride, project_valid_depth_only=False)
    assert len(full) == (w // stride) * (h // stride)
    np.testing.assert_array_equal(full[keep], p)
    assert np.all(np.isnan(full[~keep]))


def test_cutoff_colours_and_nan_rows():
    w, h = 19, 13
    rng = np.random.default_rng(9)
    depth = rng.uniform(0.2, 4.0, (h, w)).astype(np.float32)
    depth[3, 4] = 0
    depth[5, 6] = np.inf
    depth[7, 8] = np.nan
    depth[2, 2] = np.float32(2.0)
    rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    gray = rng.uniform(0, 1, (h, w)).astype(np.float32)
    K = K_of(w, h)
    keep = (depth > 0) & np.isfinite(depth) & (depth < 2.0)
    p, _, c = D.depth_to_points(depth, K, color=rgb, depth_cutoff=2.0)
    assert len(p) == np.count_nonzero(keep) and not keep[2, 2]
    np.testing.assert_array_equal(c, rgb[keep].astype(np.float32) / np.float32(255))
    _, _, g = D.depth_to_points(depth, K, color=gray, depth_cutoff=-1.0)
    keep_all = (depth > 0) & np.isfinite(depth)
    np.testing.assert_array_equal(g, np.repeat(gray[keep_all][:, None], 3, 1))
    fp, fn, fc = D.depth_to_points(depth, K, color=rgb, depth_cutoff=2.0, compute_normals=True, project_valid_depth_only=False)
    assert len(fp) == w * h
    flat = keep.reshape(-1)
    for a in (fp, fn, fc):
        assert np.all(np.isnan(a[~flat])) and np.all(np.isfinite(a[flat]))
    np.testing.assert_array_equal(fp[flat], p)
