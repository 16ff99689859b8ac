"""TriangleMesh's ComputeEdgeList, filters, GetSurfaceArea and SamplePointsUniformly through the C++ facade
(tests/cpp/facade_mesh_ops.cpp): compiles and links with plain g++ (CPU); on the GPU its known answers hold and every
result on a TSDF sphere mesh with normals and colours equals the Python path's bit for bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_mesh_ops_compiles_and_links():
    exe = build_facade("facade_mesh_ops")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_mesh_ops_match_the_python_path():
    import cupoch_b200 as cph
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    G, I = cph.geometry, cph.integration
    S = G.FilterScope
    exe = build_facade("facade_mesh_ops")
    w, h = 96, 72
    cams = ring_cameras(4, w, h)
    vol = I.UniformTSDFVolume(2.0, 96, 0.06, I.TSDFVolumeColorType.RGB8)
    rng = np.random.default_rng(8)
    for K, E in cams:
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)), G.Image(d16),
                                                     1000.0, 100.0, False)
        vol.integrate(im, cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    mesh = vol.extract_triangle_mesh()
    mesh.compute_vertex_normals()
    mesh.triangle_normals = None
    v, vn, vc, t = mesh.vertices.cpu(), mesh.vertex_normals.cpu(), mesh.vertex_colors.cpu(), mesh.triangles.cpu()
    assert len(t) > 100
    mesh.compute_edge_list()
    sh = mesh.filter_sharpen(3, 0.2, S.All)
    tb = mesh.filter_smooth_taubin(10, 0.5, -0.53, S.Normal)
    areas = cph.utility.DeviceArray((len(t),), np.float32)
    total = mesh._surface_area(areas)
    pc = mesh.sample_points_uniformly(12345)
    pt = mesh.sample_points_uniformly(777, True)
    want = {"edges": mesh.edge_list.cpu(), "sharpen_v": sh.vertices.cpu(), "sharpen_n": sh.vertex_normals.cpu(),
            "sharpen_c": sh.vertex_colors.cpu(), "simple_v": mesh.filter_smooth_simple(5, S.Color).vertex_colors.cpu(),
            "laplacian_v": mesh.filter_smooth_laplacian(10, 0.5, S.Vertex).vertices.cpu(), "taubin_n": tb.vertex_normals.cpu(),
            "taubin_v": tb.vertices.cpu(), "area": np.append(areas.cpu(), np.float32(total)), "sample_p": pc.points.cpu(),
            "sample_n": pc.normals.cpu(), "sample_c": pc.colors.cpu(), "sample_tn": pt.normals.cpu()}
    with tempfile.TemporaryDirectory() as d:
        np.concatenate([v, vn, vc]).astype(np.float32).tofile(os.path.join(d, "mesh.f32"))
        t.astype(np.int32).tofile(os.path.join(d, "mesh.i32"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        for name, a in want.items():
            a = np.ascontiguousarray(a)
            got = np.fromfile(os.path.join(d, "out_%s.%s" % (name, "i32" if name == "edges" else "f32")), a.dtype).reshape(a.shape)
            np.testing.assert_array_equal(got.view(np.uint32), a.view(np.uint32), err_msg=name)
