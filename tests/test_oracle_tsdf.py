"""CPU: the UniformTSDFVolume restatement (oracle/tsdf.c) -- the checker of csrc/tsdf.cu.

- The reference test's known answers on its five real RGB-D frames (tests/golden/tsdf_rgbd_known.npz): 2227 points
  with their normal sum and 4488 band voxels with their colour sum.  The reference's colour sum of ExtractPointCloud is
  not checked: it needs the frames' JPEG colours as the reference's libjpeg decodes them.
- Hand-worked single-voxel and single-ray cases: the int-truncated depth_trunc, the safe_width edge, the band edges
  +-0.98, the crossing interpolation and its (x, y, z, axis) order, the zero-gradient normal.
- The deviations: Reset restores the initial voxels, ExtractPointCloud is sized by its crossings, Raycast enters the grid
  on the box of the cells it samples (also along axis-aligned rays and from a camera on the grid's high side).
- A float64 restatement of Integrate, at an even resolution and at an odd one with an origin off the voxel lattice: the
  voxels whose update decision differs are listed with their margins, which must stay within a stated bound.
  ExtractPointCloud and Raycast are checked against their float64 restatements (cupoch_b200/testing/tsdf64.py) and
  against analytic planar and spherical fields in test_oracle_tsdf64.py; on the GPU all of them are checked against
  this oracle bit for bit."""
import os

import numpy as np

from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import tsdf_py as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsdf_rgbd_known.npz")
PRIMESENSE = np.float32([[525, 0, 319.5], [0, 525, 239.5], [0, 0, 1]])


def test_reference_known_answers_on_real_frames():
    g = np.load(GOLDEN)
    length, res, trunc, scale, dtrunc = g["setup"]
    vol = T.Volume(length, int(res), trunc, T.RGB8)
    for i in range(5):
        vol.integrate(T.depth_to_float(g["depth"][i], scale, dtrunc), np.zeros((480, 640, 3), np.uint8), PRIMESENSE,
                      g["extrinsics"][i])
    p, n, c = vol.extract_point_cloud()
    assert len(p) == int(g["points_count"]) == 2227 and len(c) == 2227
    assert np.all(np.abs(n.astype(np.float64).sum(0) - g["normal_sum"]) <= g["tolerance"])
    vp, vc = vol.extract_voxel_point_cloud()
    assert len(vp) == int(g["voxel_count"]) == 4488
    assert np.all(np.abs(vc.astype(np.float64).sum(0) - g["voxel_color_sum"]) <= g["tolerance"])


def test_depth_trunc_and_scale_are_truncated_to_int():
    d = np.array([[1999, 2000, 2499, 2500, 0, 65535]], np.uint16)
    got = T.depth_to_float(d, 1000.7, 2.5)  # int(1000.7) = 1000, int(2.5) = 2: cut at 2 m, >= truncates
    assert got.tolist() == [[np.float32(1999) / np.float32(1000), 0, 0, 0, 0, 0]]
    assert T.depth_to_float(d, 1000.0, 100.0)[0, 5] == np.float32(65535) / np.float32(1000)
    # 8-bit depth is scaled by 1/255 first (CreateFloatImage)
    assert T.depth_to_float(np.array([[255]], np.uint8), 1.0, 5.0)[0, 0] == np.float32(255) * np.float32(1 / 255)


def test_intensity_weights():
    c = np.array([[[255, 0, 0], [0, 255, 0], [0, 0, 255], [10, 20, 30]]], np.uint8)
    got = T.intensity(c)[0]
    w = np.float32([0.299, 0.587, 0.114])
    want = [np.float32(w[0] * np.float32(255)) * np.float32(1 / 255), np.float32(w[1] * np.float32(255)) * np.float32(1 / 255),
            np.float32(w[2] * np.float32(255)) * np.float32(1 / 255)]
    assert np.array_equal(got[:3], np.float32(want))
    assert abs(got[3] - (0.299 * 10 + 0.587 * 20 + 0.114 * 30) / 255) < 1e-6


def one_camera(w=4, h=3, f=2.0):
    """a camera at the origin looking along +z: K, identity extrinsic"""
    return np.float32([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]]), np.eye(4, dtype=np.float32)


def test_integrate_single_voxel_and_safe_width_edge():
    # res 2, length 2: voxel centres at -0.5 / 0.5; shift the origin so voxel (1, 1, 1) sits at (0, 0, 2)
    vol = T.Volume(2.0, 2, 0.5, T.NO_COLOR, origin=(-0.5, -0.5, 1.5))
    K, E = one_camera()
    depth = np.full((3, 4), 2.1, np.float32)
    vol.integrate(depth, None, K, E)
    i = 7  # (1, 1, 1)
    # u = 0 * f / 2 + 1.5 + 0.5 = 2 -> pixel (2, 1); multiplier sqrt(((2 - 1.5) / 2)^2 + 0 + 1)
    mult = np.sqrt(np.float32(0.25) ** 2 + np.float32(1))
    sdf = (np.float32(2.1) - np.float32(2.0)) * np.float32(mult)
    assert vol.tw[i, 1] == 1 and vol.tw[i, 0] == min(np.float32(1), sdf * np.float32(1 / 0.5))
    # voxel (0, 0, 0) at (-1, -1, 1): u = -1 * 2 / 1 + 2 = 0 < 0.0001 -> outside, untouched
    assert vol.tw[0].tolist() == [0, 0]
    # the safe_width edge: u must stay below width - 0.0001
    K2 = np.float32([[2, 0, 3.4999], [0, 2, 1], [0, 0, 1]])  # voxel (1, 1, 1): u = 3.4999 + 0.5 = 3.9999 < 3.9999? no
    v2 = T.Volume(2.0, 2, 0.5, T.NO_COLOR, origin=(-0.5, -0.5, 1.5))
    v2.integrate(depth, None, K2, E)
    assert v2.tw[7, 1] == 0
    K3 = np.float32([[2, 0, 3.4997], [0, 2, 1], [0, 0, 1]])
    v3 = T.Volume(2.0, 2, 0.5, T.NO_COLOR, origin=(-0.5, -0.5, 1.5))
    v3.integrate(depth, None, K3, E)
    assert v3.tw[7, 1] == 1


def test_integrate_skips_behind_the_truncation_and_zero_depth():
    K, E = one_camera()
    # sdf = (d - 2) * 1.0308 (the pixel's camera-distance multiplier): -0.5 / 1.0308 = -0.485 is the limit
    for d, updated in ((2.0 - 0.49, False), (2.0 - 0.48, True), (0.0, False), (-1.0, False)):
        vol = T.Volume(2.0, 2, 0.5, T.NO_COLOR, origin=(-0.5, -0.5, 1.5))
        vol.integrate(np.full((3, 4), d, np.float32), None, K, E)
        assert (vol.tw[7, 1] == 1) == updated, d


def test_weighted_running_means_and_rgb_units():
    K, E = one_camera()
    vol = T.Volume(2.0, 2, 0.5, T.RGB8, origin=(-0.5, -0.5, 1.5))
    col = np.zeros((3, 4, 3), np.uint8)
    col[1, 2] = (200, 100, 50)
    vol.integrate(np.full((3, 4), 2.1, np.float32), col, K, E)
    assert vol.col[:, 7].tolist() == [200, 100, 50]  # (1 * 0 + c) / 1: the initial (1, 1, 1) has weight 0
    col[1, 2] = (100, 0, 250)
    vol.integrate(np.full((3, 4), 2.1, np.float32), col, K, E)
    assert vol.col[:, 7].tolist() == [150, 50, 150] and vol.tw[7, 1] == 2
    assert vol.col[:, 0].tolist() == [1, 1, 1]


def test_band_edges():
    vol = T.Volume(4.0, 4, 1.0)
    fs = [0.98, np.nextafter(np.float32(0.98), np.float32(0)), -0.98, np.nextafter(np.float32(-0.98), np.float32(-1)), 0.0]
    for k, f in enumerate(fs):
        vol.tw[k] = (f, 1.0)
    vol.tw[5] = (0.5, 0.0)  # weight 0: never in the band
    keys, cols, _, _ = vol.extract_voxel_grid()
    assert keys.tolist() == [[0, 0, 1], [0, 0, 2], [0, 1, 0]]
    assert cols[:, 0].tolist() == [np.float32((np.float64(np.float32(f)) + 1) * 0.5) for f in (fs[1], -0.98, 0.0)]
    # voxel centres: vl (k - res / 2) + vl / 2 + origin
    p, _ = vol.extract_voxel_point_cloud()
    assert p.tolist() == [[-1.5, -1.5, -0.5], [-1.5, -1.5, 0.5], [-1.5, -0.5, -1.5]]


def test_crossing_interpolation_order_and_interior_rule():
    vol = T.Volume(6.0, 6, 1.0)
    res = 6

    def put(x, y, z, f):
        vol.tw[(x * res + y) * res + z] = (f, 1.0)
    put(2, 2, 2, 0.5)
    put(3, 2, 2, -0.25)  # x crossing
    put(2, 2, 3, -0.5)   # z crossing
    put(2, 3, 2, 0.4)    # same sign: none
    put(4, 2, 2, 0.5)    # (3, 2, 2) -> (4, 2, 2) is another x crossing
    put(0, 2, 2, -0.5)   # x = 0 is not interior: (0) -> (1) is never tested
    p, n, _ = vol.extract_point_cloud()
    # rows in (x, y, z, axis) order: (2,2,2) axis 0, (2,2,2) axis 2, (3,2,2) axis 0
    assert len(p) == 3
    # axis 0 of (2,2,2): p0 = 2.5, p1 = 3.5, r0 = 0.5, r1 = 0.25 -> (2.5 * 0.25 + 3.5 * 0.5) / 0.75, then - 3 (res / 2 vl)
    assert p[0].tolist() == [np.float32(np.float32(2.375) / np.float32(0.75)) - 3, -0.5, -0.5]
    assert p[1].tolist() == [-0.5, -0.5, 0.0]
    assert p[2, 0] == np.float32(np.float32(3.5 * 0.5 + 4.5 * 0.25) / np.float32(0.75)) - 3
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6)


def test_zero_gradient_normal_is_left_unnormalised():
    """Eigen's normalized() (>= 3.3) returns the vector unchanged when its squared norm is not > 0, instead of dividing by
    0.  A crossing between (4,3,3) = 0.5 and (5,3,3) = -1e-30 sits at the centre of voxel 5; its two x samples at
    p -+ 0.99 vl read 0.5 (1 - r) + f1 r and f1 r + 0.5 (1 - r) with the same r, so the x difference is exactly 0, and the
    y / z differences are ~1e-37, whose squares underflow: the normal is returned as computed, not normalised."""
    res = 10
    vol = T.Volume(10.0, res, 1.0)
    idx = lambda x, y, z: (x * res + y) * res + z  # noqa: E731
    vol.tw[idx(4, 3, 3)], vol.tw[idx(5, 3, 3)], vol.tw[idx(6, 3, 3)] = (0.5, 1), (-1e-30, 1), (0.5, 0)
    p, n, _ = vol.extract_point_cloud()
    assert p.tolist() == [[0.5, -1.5, -1.5]]
    assert n[0, 0] == 0 and 0 < -n[0, 1] < 1e-30 and n[0, 1] == n[0, 2]
    assert np.float32(n[0, 1]) * np.float32(n[0, 1]) == 0  # the squared norm underflows to 0


def sphere_volume(res=64, views=6, w=96, h=72, trunc=0.08):
    vol = T.Volume(2.0, res, trunc)
    cams = ring_cameras(views, w, h)
    for K, E in cams:
        vol.integrate(sphere_depth(K, E, w, h, 0.6), None, K, E)
    return vol, cams


def test_reset_restores_the_initial_voxels():
    vol = T.Volume(2.0, 16, 0.2, T.RGB8)
    K, E = ring_cameras(1, 32, 24)[0]
    vol.integrate(sphere_depth(K, E, 32, 24, 0.6), np.full((24, 32, 3), 9, np.uint8), K, E)
    assert vol.tw[:, 1].any()
    vol.reset()
    assert not vol.tw.any() and np.all(vol.col == 1)
    assert len(vol.extract_point_cloud()[0]) == 0 and len(vol.extract_voxel_point_cloud()[0]) == 0


def test_point_output_is_sized_by_crossings_not_band_voxels():
    """a checkerboard of +-0.5 makes every interior band voxel emit three points: the reference's output, sized by the
    band voxels, would be overrun three times over"""
    res = 8
    vol = T.Volume(8.0, res, 1.0)
    x, y, z = np.meshgrid(np.arange(res), np.arange(res), np.arange(res), indexing="ij")
    vol.tw[:, 0] = np.where((x + y + z) % 2 == 0, 0.5, -0.5).reshape(-1)
    vol.tw[:, 1] = 1.0
    p, n, _ = vol.extract_point_cloud()
    band = len(vol.extract_voxel_point_cloud()[0])
    inner = res - 2
    # axis i of interior voxel k emits while k_i + 1 <= res - 2
    assert len(p) == 3 * inner * inner * (inner - 1) and len(p) > band == res ** 3


def test_raycast_enters_on_the_grids_real_box():
    """camera 2.5 in front of a sphere of radius 0.6 at the centre of a [-1, 1]^3 grid, looking along +x through pixel
    (16, 12) exactly, so two direction components are 0: the hit is the sphere's front at x = -0.6.  The reference's
    box [0, length]^3 in origin-relative coordinates would start the march at t = 2.5, at x = 0, past that surface."""
    vol, _ = sphere_volume()
    K = np.float32([[40, 0, 16], [0, 40, 12], [0, 0, 1]])
    E = np.zeros((4, 4), np.float32)
    E[0, 1] = E[1, 2] = E[2, 0] = E[3, 3] = 1  # camera x, y, z = world y, z, x
    E[2, 3] = 2.5  # eye at (-2.5, 0, 0)
    p, n, _ = vol.raycast(K, E, 33, 25, 0.08, False)
    c = p[12 * 33 + 16]
    assert c[1] == 0 and c[2] == 0 and abs(c[0] + 0.6) < 2.0 / 64
    assert n[12 * 33 + 16, 0] < -0.99
    t_ref_entry = (0.0 - (-2.5)) / 1.0  # GetMinTime with the origin-relative camera x = -2.5 and direction +x
    assert -2.5 + t_ref_entry > -0.6
    # every hit lies on the sphere within a voxel; project_valid_depth_only keeps exactly the hit rows, in order
    hp, _, _ = vol.raycast(K, E, 33, 25, 0.08, True)
    assert np.array_equal(hp, p[np.isfinite(p[:, 0])]) and len(hp) > 100
    assert np.all(np.abs(np.linalg.norm(hp, axis=1) - 0.6) < 2.0 / 64)


def integrate_vs_float64(res, origin=(0.0, 0.0, 0.0)):
    """Integrate restated in float64 on 4 sphere views: the update decisions that differ from the float32 restatement
    are listed with their margins -- how far the float64 quantity was from the rule's threshold (z <= 0, the image
    bounds, sdf > -trunc) -- which stay below 1e-5; the tsdf of the voxels both update agrees to 1e-4."""
    length, trunc, w, h = 2.0, 0.1, 80, 60
    vol = T.Volume(length, res, trunc, origin=origin)
    vl = length / res
    hres = res // 2
    o = np.asarray(origin, np.float32).astype(np.float64)
    k = (np.arange(res) - hres) * vl + vl / 2
    X, Y, Z = np.meshgrid(k + o[0], k + o[1], k + o[2], indexing="ij")
    P = np.stack([X, Y, Z], -1).reshape(-1, 3)
    tsdf64, w64 = np.zeros(len(P)), np.zeros(len(P))
    differing = []
    for K, E in ring_cameras(4, w, h):
        d = sphere_depth(K, E, w, h, 0.6)
        before = vol.tw[:, 1].copy()
        vol.integrate(d, None, K, E)
        upd32 = vol.tw[:, 1] != before
        E64, K64 = E.astype(np.float64), K.astype(np.float64)
        cam = P @ E64[:3, :3].T + E64[:3, 3]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = cam[:, 0] * K64[0, 0] / cam[:, 2] + K64[0, 2] + 0.5
            v = cam[:, 1] * K64[1, 1] / cam[:, 2] + K64[1, 2] + 0.5
        inside = (cam[:, 2] > 0) & (u >= 1e-4) & (u < w - 1e-4) & (v >= 1e-4) & (v < h - 1e-4)
        ui, vi = np.where(inside, np.floor(u), 0).astype(int), np.where(inside, np.floor(v), 0).astype(int)
        dd = d[vi, ui].astype(np.float64)
        mult = np.sqrt(((ui - K64[0, 2]) / K64[0, 0]) ** 2 + ((vi - K64[1, 2]) / K64[1, 1]) ** 2 + 1)
        sdf = (dd - cam[:, 2]) * mult
        upd64 = inside & (dd > 0) & (sdf > -trunc)
        t = np.minimum(1.0, sdf / trunc)
        tsdf64 = np.where(upd64, (tsdf64 * w64 + t) / (w64 + 1), tsdf64)
        w64 = np.where(upd64, w64 + 1, w64)
        for i in np.nonzero(upd32 != upd64)[0]:
            margin = min(abs(sdf[i] + trunc), abs(u[i] - 1e-4), abs(u[i] - (w - 1e-4)), abs(v[i] - 1e-4), abs(v[i] - (h - 1e-4)),
                         abs(u[i] - np.round(u[i])), abs(v[i] - np.round(v[i])))
            differing.append((int(i), float(margin)))
    assert all(m < 1e-5 for _, m in differing), differing
    both = (vol.tw[:, 1] == w64) & (w64 > 0)
    assert both.sum() > 1000 and len(differing) < 0.001 * both.sum()
    assert np.max(np.abs(vol.tw[both, 0] - tsdf64[both])) < 1e-4


def test_integrate_against_a_float64_restatement():
    """a 48^3 volume at the origin"""
    integrate_vs_float64(48)


def test_integrate_against_a_float64_restatement_at_odd_res_and_an_offset_origin():
    """47^3 (res / 2 rounds down) with an origin off the voxel lattice"""
    integrate_vs_float64(47, (0.0123, -0.0311, 0.0057))


def test_raycast_from_a_camera_on_the_high_side_hits():
    """a camera on +x enters through the grid's high x face; the first sample, one voxel in, must land in a cell the
    march reads (below res - 1), so the entry box ends at cell res - 1.  Nearly every pixel that saw the sphere hits."""
    w, h = 160, 120
    K, E = ring_cameras(1, w, h)[0]  # eye at (2.5, 0, 0)
    vol = T.Volume(2.0, 128, 0.06)
    d = sphere_depth(K, E, w, h, 0.6)
    vol.integrate(d, None, K, E)
    p, _, _ = vol.raycast(K, E, w, h, 0.06, False)
    assert np.isfinite(p[:, 0]).sum() >= 0.95 * (d > 0).sum()
