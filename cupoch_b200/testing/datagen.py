"""Synthetic clouds of SURVEY.md section 8d (seeded numpy PCG64, float32).  Shared by tests/ and bench.py."""
import numpy as np


def rot_xyz(rx_deg, ry_deg, rz_deg):
    rx, ry, rz = np.deg2rad([rx_deg, ry_deg, rz_deg])
    Rx = np.array([[1, 0, 0], [0, np.cos(rx), -np.sin(rx)], [0, np.sin(rx), np.cos(rx)]])
    Ry = np.array([[np.cos(ry), 0, np.sin(ry)], [0, 1, 0], [-np.sin(ry), 0, np.cos(ry)]])
    Rz = np.array([[np.cos(rz), -np.sin(rz), 0], [np.sin(rz), np.cos(rz), 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def gt_transform(angles=(-2.0, 3.0, 5.0), t=(0.02, -0.01, 0.015)):
    """T_gt = Rz(5) Ry(3) Rx(-2), t = (0.02,-0.01,0.015)  (section 8d, config 1)."""
    T = np.eye(4)
    T[:3, :3] = rot_xyz(*angles)
    T[:3, 3] = t
    return T


def uniform_cube(n, seed, lo=(0, 0, 0), hi=(1, 1, 1)):
    rng = np.random.Generator(np.random.PCG64(seed))
    p = rng.random((n, 3), dtype=np.float32)
    return (np.asarray(lo, np.float32) + p * (np.asarray(hi, np.float32) - np.asarray(lo, np.float32))).astype(np.float32)


def unit_normals(n, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    v = rng.standard_normal((n, 3)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v.astype(np.float32)


def surface(n, seed, extent=1.0):
    """z = 0.1 sin(4 pi x) cos(4 pi y), x,y ~ U[0,extent); analytic unit normals (config 2)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    xy = rng.random((n, 2)) * extent
    x, y = xy[:, 0], xy[:, 1]
    z = 0.1 * np.sin(4 * np.pi * x) * np.cos(4 * np.pi * y)
    dzdx = 0.4 * np.pi * np.cos(4 * np.pi * x) * np.cos(4 * np.pi * y)
    dzdy = -0.4 * np.pi * np.sin(4 * np.pi * x) * np.sin(4 * np.pi * y)
    nrm = np.stack([-dzdx, -dzdy, np.ones_like(x)], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return np.stack([x, y, z], 1).astype(np.float32), nrm.astype(np.float32)


def plane_scene(n, seed, noise=0.003):
    """SegmentPlane scene: 50 % on a noisy ground z = 0 (axis-aligned, the case where the refit cancels worst), 20 % on a
    tilted wall, 30 % clutter in [-2, 2]^2 x [0, 2], rows shuffled."""
    rng = np.random.Generator(np.random.PCG64(seed))
    ng, nw = n // 2, n // 5
    g = np.column_stack([rng.uniform(-2, 2, (ng, 2)), rng.normal(0, noise, ng)])
    uv = rng.uniform(0, 2, (nw, 2))
    w = np.column_stack([uv[:, 0] - 1, 1.5 + 0.3 * uv[:, 1], uv[:, 1]]) + rng.normal(0, noise, (nw, 3))
    c = np.column_stack([rng.uniform(-2, 2, (n - ng - nw, 2)), rng.uniform(0, 2, n - ng - nw)])
    p = np.concatenate([g, w, c]).astype(np.float32)
    return p[rng.permutation(n)]


def texture(p, seed=None, noise=0.0):
    """smooth colour field in [0,1]^3 (config 5)."""
    x, y = p[:, 0].astype(np.float64), p[:, 1].astype(np.float64)
    c = np.stack([0.5 + 0.4 * np.sin(7 * x) * np.cos(5 * y), 0.5 + 0.4 * np.cos(3 * x + 2 * y),
                  0.5 + 0.4 * np.sin(4 * y - x)], 1)
    if noise > 0:
        rng = np.random.Generator(np.random.PCG64(seed))
        c = c + rng.normal(0, noise, c.shape)
    return np.clip(c, 0, 1).astype(np.float32)


def make_source(target, T_gt, perm_seed, noise_seed, sigma, attrs=()):
    """source = target[perm] moved by T_gt^-1 plus N(0, sigma^2) noise; attrs are permuted and rotated alike."""
    n = len(target)
    perm = np.random.Generator(np.random.PCG64(perm_seed)).permutation(n)
    Ti = np.linalg.inv(T_gt)
    p = target[perm].astype(np.float64) @ Ti[:3, :3].T + Ti[:3, 3]
    if sigma > 0:
        p = p + np.random.Generator(np.random.PCG64(noise_seed)).normal(0, sigma, p.shape)
    out = [p.astype(np.float32)]
    for a, is_vec in attrs:
        b = a[perm]
        if is_vec:
            b = (b.astype(np.float64) @ Ti[:3, :3].T)
        out.append(np.ascontiguousarray(b, np.float32))
    return out if len(out) > 1 else out[0]


def ring_cameras(views, w, h, radius=2.5, f=None):
    """carving views: cameras on a tilted ring of the given radius around the origin, each looking at it.  -> a list of
    (K [3, 3], world-to-camera E [4, 4]) float32 pairs; f defaults to 0.9 w"""
    f = f or 0.9 * w
    K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], np.float32)
    out = []
    for i in range(views):
        a = 2 * np.pi * i / views
        eye = np.array([radius * np.cos(a), radius * np.sin(a), 0.6 * np.sin(3 * a)])
        zc = -eye / np.linalg.norm(eye)
        xc = np.cross(zc, [0, 0, 1.0])
        xc /= np.linalg.norm(xc)
        R = np.stack([xc, np.cross(zc, xc), zc])
        E = np.eye(4, dtype=np.float32)
        E[:3, :3] = R
        E[:3, 3] = -R @ eye
        out.append((K, E))
    return out


def sphere_depth(K, E, w, h, radius):
    """analytic depth map (camera z, float32 [h, w]) of a sphere of the given radius at the world origin seen through
    K and the world-to-camera E; 0 where the ray misses"""
    Ki = np.linalg.inv(np.asarray(K, np.float64))
    uu, vv = np.meshgrid(np.arange(w), np.arange(h))
    rays = np.stack([uu, vv, np.ones_like(uu)], -1).reshape(-1, 3) @ Ki.T  # camera rays with z = 1
    R, t = np.asarray(E, np.float64)[:3, :3], np.asarray(E, np.float64)[:3, 3]
    c = -R.T @ t  # camera centre in the world
    dw = rays @ R  # world directions (R^T d)
    a = np.sum(dw * dw, 1)
    b = 2 * dw @ c
    cc = c @ c - radius * radius
    disc = b * b - 4 * a * cc
    s = (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a)
    return np.where(disc > 0, s, 0).reshape(h, w).astype(np.float32)
