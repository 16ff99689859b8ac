"""GPU: TriangleMesh.compute_edge_list, the four filters, get_surface_area and sample_points_uniformly (csrc/mesh.cu)
against oracle/mesh_ops.c bit for bit: the reference's fixtures, meshes extracted from TSDF sphere views and from the
five real frames, and random meshes with isolated vertices, a repeated-vertex triangle and duplicate positions.  Also
every FilterScope against every attribute combination, iterations 0 / 1 / 100, user-set and rejected edge lists,
repeats, the launch count per pass, and point-to-plane ICP on two samples of one mesh."""
import itertools
import json
import os

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import cupoch_b200 as cph
from cupoch_b200 import _lib
from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
from oracle import mesh_ops_py as M, tsdf_py as T

G, CAM, I = cph.geometry, cph.camera, cph.integration
CT = I.TSDFVolumeColorType
S = G.FilterScope
HERE = os.path.dirname(os.path.abspath(__file__))
MASK = {S.All: 7, S.Vertex: 1, S.Normal: 2, S.Color: 4}


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def sphere_mesh(res=128, ct=CT.RGB8, views=8):
    w, h = 160, 120
    vol = I.UniformTSDFVolume(2.0, res, 0.06, ct)
    rng = np.random.default_rng(res)
    for K, E in ring_cameras(views, w, h, 2.5):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)), G.Image(d16),
                                                     1000.0, 100.0, ct == CT.Gray32)
        vol.integrate(im, CAM.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    return vol.extract_triangle_mesh()


def real_mesh():
    g = np.load(os.path.join(HERE, "golden", "tsdf_rgbd_known.npz"))
    K = CAM.PinholeCameraIntrinsic(CAM.PinholeCameraIntrinsicParameters.PrimeSenseDefault)
    vol = I.UniformTSDFVolume(8.0, 200, 0.04, CT.RGB8)
    rng = np.random.default_rng(5)
    for i in range(5):
        color = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(color), G.Image(g["depth"][i]), 1000.0, 4.0, False)
        vol.integrate(im, K, g["extrinsics"][i])
    return vol.extract_triangle_mesh()


def random_mesh(seed, nv=3000, nt=5000):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(nv, 3)).astype(np.float32)
    pool = np.setdiff1d(np.arange(nv), [0, 17, nv - 1])
    t = np.stack([rng.choice(pool, 3, replace=False) for _ in range(nt)]).astype(np.int32)
    t[3] = (t[3, 0], t[3, 0], t[3, 2])
    v[t[5, 1]] = v[t[5, 0]]
    m = G.TriangleMesh(v, t)
    m.vertex_normals = rng.normal(size=(nv, 3)).astype(np.float32)
    m.vertex_colors = rng.uniform(0, 1, (nv, 3)).astype(np.float32)
    return m


@pytest.fixture(scope="module")
def meshes():
    out = {"sphere": sphere_mesh(), "real": real_mesh(), "random": random_mesh(1)}
    out["sphere"].compute_vertex_normals()
    out["real"].compute_vertex_normals()
    return out


def attrs(m):
    return (m.vertices.cpu(), m.vertex_normals.cpu() if m.has_vertex_normals() else None,
            m.vertex_colors.cpu() if m.has_vertex_colors() else None)


def with_attrs(m, normals, colors):
    """a copy of m's vertices and triangles, with its normals / colours only when asked"""
    out = G.TriangleMesh(m.vertices.cpu(), m.triangles.cpu())
    if normals:
        out.vertex_normals = m.vertex_normals.cpu()
    if colors:
        out.vertex_colors = m.vertex_colors.cpu()
    return out


def run(m, kind, it, scope, c0, c1):
    f = {M.SHARPEN: lambda: m.filter_sharpen(it, c0, scope), M.SIMPLE: lambda: m.filter_smooth_simple(it, scope),
         M.LAPLACIAN: lambda: m.filter_smooth_laplacian(it, c0, scope),
         M.TAUBIN: lambda: m.filter_smooth_taubin(it, c0, c1, scope)}
    return f[kind]()


def check_filter(m, kind, it, scope, c0=0.5, c1=-0.53):
    out = run(m, kind, it, scope, c0, c1)
    v, n, c = attrs(m)
    rv, rn, rc = M.filter_mesh(kind, it, M.edge_list(m.triangles.cpu(), len(v)), v, n, c, MASK[scope], c0, c1)
    gv, gn, gc = attrs(out)
    assert same(gv, rv) and (n is None) == (gn is None) and (c is None) == (gc is None)
    assert n is None or same(gn, rn)
    assert c is None or same(gc, rc)
    assert same(out.triangles.cpu(), m.triangles.cpu()) and out.triangle_normals is None
    return out


def test_golden_fixtures():
    with open(os.path.join(HERE, "golden", "mesh_ops_known.json")) as f:
        g = json.load(f)
    e = g["edge_list"]
    m = G.TriangleMesh(np.float32(e["vertices"]), np.int32(e["triangles"]))
    assert not m.has_edge_list()
    assert np.array_equal(m.compute_edge_list().edge_list.cpu(), np.int32(e["edges"])) and m.has_edge_list()
    f = g["filters"]
    cur = {}
    for st in f["steps"]:
        k, a = st["filter"], st["args"]
        m = cur.get(k) or G.TriangleMesh(np.float32(f["vertices"]), np.int32(f["triangles"]))
        it = a["number_of_iterations"]
        out = {"sharpen": lambda: m.filter_sharpen(it, a["strength"]), "simple": lambda: m.filter_smooth_simple(it),
               "laplacian": lambda: m.filter_smooth_laplacian(it, **{"lambda": a["lambda"]}),
               "taubin": lambda: m.filter_smooth_taubin(it, a["lambda"], a["mu"])}[k]()
        np.testing.assert_allclose(out.vertices.cpu(), np.float32(st["vertices"]), atol=g["tolerance"])
        kind = {"sharpen": M.SHARPEN, "simple": M.SIMPLE, "laplacian": M.LAPLACIAN, "taubin": M.TAUBIN}[k]
        want = M.filter_mesh(kind, it, out.edge_list.cpu(), m.vertices.cpu(), c0=a.get("strength", a.get("lambda", 0.0)),
                             c1=a.get("mu", 0.0))[0]
        assert same(out.vertices.cpu(), want) and out.has_edge_list()
        cur[k] = out
    s = g["sample_points_uniformly"]
    m = G.TriangleMesh(np.float32(s["vertices"]), np.int32(s["triangles"]))
    pc = m.sample_points_uniformly(100)
    assert len(pc.points) == 100 and not pc.has_normals() and not pc.has_colors()
    m.vertex_colors, m.vertex_normals = np.float32(s["vertex_colors"]), np.float32(s["vertex_normals"])
    pc = m.sample_points_uniformly(100)
    tol = g["tolerance"]  # interpolated attributes: a + b + c is 1 only to rounding
    np.testing.assert_allclose(pc.colors.cpu(), np.float32([[1, 0, 0]] * 100), atol=tol)
    np.testing.assert_allclose(pc.normals.cpu(), np.float32([[0, 1, 0]] * 100), atol=tol)
    assert not m.has_triangle_normals()
    pc = m.sample_points_uniformly(100, True)
    assert m.has_triangle_normals() and np.all(pc.normals.cpu() == np.float32([0, 0, 1]))
    np.testing.assert_allclose(pc.colors.cpu(), np.float32([[1, 0, 0]] * 100), atol=tol)
    m.vertex_normals = np.zeros((0, 3), np.float32)
    pc = m.sample_points_uniformly(100, True)
    assert len(pc.normals) == 100 and np.all(pc.normals.cpu() == np.float32([0, 0, 1]))
    p, nr, c, _ = M.sample_points_uniformly(s["vertices"], s["triangles"], 100, None, m.triangle_normals.cpu(), s["vertex_colors"])
    assert same(pc.points.cpu(), p) and same(pc.normals.cpu(), nr) and same(pc.colors.cpu(), c)
    with pytest.raises(ValueError):
        G.TriangleMesh().sample_points_uniformly(100)


@pytest.mark.parametrize("name", ["sphere", "real", "random"])
def test_edge_list_matches_oracle(meshes, name):
    m = meshes[name]
    e = G.TriangleMesh(m.vertices.cpu(), m.triangles.cpu()).compute_edge_list().edge_list.cpu()
    assert same(e, M.edge_list(m.triangles.cpu(), len(m.vertices)))


@pytest.mark.parametrize("name", ["sphere", "real", "random"])
@pytest.mark.parametrize("kind", [M.SHARPEN, M.SIMPLE, M.LAPLACIAN, M.TAUBIN])
def test_filters_match_oracle_for_every_scope_and_attribute_set(meshes, name, kind):
    base = meshes[name]
    c0 = 0.002 if kind == M.SHARPEN else 0.5  # Sharpen amplifies: keep 100 iterations finite on a random mesh's degrees
    for normals, colors in itertools.product((False, True), repeat=2):
        m = with_attrs(base, normals, colors)
        for scope in (S.All, S.Vertex, S.Normal, S.Color):
            check_filter(m, kind, 1, scope, c0)
    m = with_attrs(base, True, True)
    for it in (0, 100):
        check_filter(m, kind, it, S.All, c0)


def test_sphere_views_at_every_colour_type():
    for ct in (CT.NoColor, CT.Gray32):
        m = sphere_mesh(96, ct, 6)
        for kind in (M.SIMPLE, M.TAUBIN):
            check_filter(m, kind, 3, S.All)


def test_user_edge_list_is_used_and_bad_ones_rejected(meshes):
    m = with_attrs(meshes["random"], True, True)
    e = M.edge_list(m.triangles.cpu(), len(m.vertices))
    sub = e[::3].copy()  # a sorted subset: the filter must follow it, not the triangles
    m.edge_list = sub
    out = m.filter_smooth_laplacian(2, 0.4)
    v, n, c = attrs(m)
    rv, rn, rc = M.filter_mesh(M.LAPLACIAN, 2, sub, v, n, c, 7, 0.4)
    assert same(out.vertices.cpu(), rv) and same(out.vertex_normals.cpu(), rn) and same(out.edge_list.cpu(), sub)
    for bad in (e[::-1].copy(), np.concatenate([e, [[len(v), 0]]]).astype(np.int32), np.concatenate([[[-1, 0]], e]).astype(np.int32)):
        m.edge_list = bad
        with pytest.raises(_lib.CphbError):
            m.filter_smooth_simple(1)
    bad_tri = G.TriangleMesh(m.vertices.cpu(), np.int32([[0, 1, len(v)]]))
    for call in (bad_tri.compute_edge_list, bad_tri.get_surface_area, lambda: bad_tri.sample_points_uniformly(10)):
        with pytest.raises(_lib.CphbError):
            call()


@pytest.mark.parametrize("name", ["sphere", "real", "random"])
def test_surface_area_matches_oracle_and_repeats(meshes, name):
    m = meshes[name]
    a = m.get_surface_area()
    want, areas = M.surface_area(m.vertices.cpu(), m.triangles.cpu())
    assert np.float32(a) == want and all(m.get_surface_area() == a for _ in range(3))
    buf = cph.utility.DeviceArray((len(m.triangles),), np.float32)
    assert m._surface_area(buf) == a and same(buf.cpu(), areas)


def test_sphere_area_is_close_to_4_pi_r2(meshes):
    a = meshes["sphere"].get_surface_area()
    # marching cubes on a 2 m / 128 grid: the mesh lies within about a voxel of the r = 0.6 sphere, and its facets
    # make it at most a few per cent larger than the smooth surface
    r, vox = 0.6, 2.0 / 128
    assert 4 * np.pi * (r - vox) ** 2 < a < 1.1 * 4 * np.pi * (r + vox) ** 2


@pytest.mark.parametrize("name", ["sphere", "real", "random"])
def test_sampling_matches_oracle(meshes, name):
    m = meshes[name]
    nt = len(m.triangles)
    for n, tri_normal in ((nt // 3, False), (100000, False), (54321, True)):
        mm = with_attrs(m, True, True)
        pc = mm.sample_points_uniformly(n, tri_normal)
        tn = mm.triangle_normals.cpu() if tri_normal else None
        if tri_normal:
            assert same(tn, G.TriangleMesh(m.vertices.cpu(), m.triangles.cpu()).compute_triangle_normals().triangle_normals.cpu())
        p, nr, c, _ = M.sample_points_uniformly(m.vertices.cpu(), m.triangles.cpu(), n, m.vertex_normals.cpu(), tn, m.vertex_colors.cpu())
        assert same(pc.points.cpu(), p) and same(pc.normals.cpu(), nr) and same(pc.colors.cpu(), c)
        again = mm.sample_points_uniformly(n, tri_normal)
        assert same(again.points.cpu(), p)
    plain = G.TriangleMesh(m.vertices.cpu(), m.triangles.cpu()).sample_points_uniformly(5000)
    assert same(plain.points.cpu(), M.sample_points_uniformly(m.vertices.cpu(), m.triangles.cpu(), 5000)[0])
    assert not plain.has_normals() and not plain.has_colors()


def test_sampling_rejects_bad_requests():
    m = G.TriangleMesh(np.float32([[0, 0, 0], [1, 0, 0], [2, 0, 0]]), np.int32([[0, 1, 2]]))
    with pytest.raises(_lib.CphbError):
        m.sample_points_uniformly(10)  # zero area
    m = G.TriangleMesh(np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]]), np.int32([[0, 1, 2]]))
    for n in (0, 2 ** 30):
        with pytest.raises(ValueError):
            m.sample_points_uniformly(n)


def test_repeats_are_bit_identical_and_the_launch_count_fixed(meshes):
    m = with_attrs(meshes["sphere"], True, True)
    m.compute_edge_list()
    L = _lib.lib()
    for kind in (M.SHARPEN, M.SIMPLE, M.LAPLACIAN, M.TAUBIN):
        counts = {}
        for it in (1, 2, 7):
            outs = []
            for _ in range(2):
                n0 = L.cphb_launch_count()
                outs.append(attrs(run(m, kind, it, S.All, 0.1, -0.11)))
                counts[it] = L.cphb_launch_count() - n0
            assert all(same(a, b) for a, b in zip(*outs))
        per_pass = 2 if kind == M.TAUBIN else 1
        assert counts[2] - counts[1] == per_pass and counts[7] - counts[1] == 6 * per_pass, counts
        setup = 3 if kind in (M.LAPLACIAN, M.TAUBIN) else 2  # check, rows (, weights)
        assert counts[1] == setup + per_pass, counts
    n0 = L.cphb_launch_count()
    m.sample_points_uniformly(1000)
    assert L.cphb_launch_count() - n0 == 4


def test_icp_recovers_a_rigid_transform_between_two_samples(meshes):
    m = meshes["sphere"]
    R = cph.registration
    a = G.TriangleMesh(m.vertices.cpu(), m.triangles.cpu()).sample_points_uniformly(60000)
    b = G.TriangleMesh(m.vertices.cpu(), m.triangles.cpu())
    # a different sample of the same surface: shift the draw sequence by sampling more points and keeping a tail
    b_pts = b.sample_points_uniformly(120000).points.cpu()[1::2]
    ang = np.deg2rad(3.0)
    Tm = np.eye(4, dtype=np.float32)
    Tm[:3, :3] = np.float32([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]])
    Tm[:3, 3] = (0.02, -0.01, 0.015)
    tgt = G.PointCloud((b_pts @ Tm[:3, :3].T + Tm[:3, 3]).astype(np.float32))
    tgt.estimate_normals(G.KDTreeSearchParamKNN(20))
    res = R.registration_icp(a, tgt, 0.1, np.eye(4), R.TransformationEstimationPointToPlane(), R.ICPConvergenceCriteria(1e-8, 1e-8, 60))
    err = np.abs(np.asarray(res.transformation, np.float64) - Tm).max()
    assert res.fitness > 0.95 and err < 2e-3, (res.fitness, err)
