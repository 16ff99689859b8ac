"""UniformTSDFVolume::ExtractTriangleMesh and TriangleMesh through the C++ facade (tests/cpp/facade_mesh.cpp): compiles
and links with plain g++ (CPU); on the GPU its known answers hold, and the mesh and normals of an RGB8 volume integrated
from four sphere views equal the Python path's (extract_triangle_mesh, compute_vertex_normals) bit for bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_mesh_compiles_and_links():
    exe = build_facade("facade_mesh")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_mesh_matches_the_python_path():
    import cupoch_b200 as cph
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    G, I = cph.geometry, cph.integration
    exe = build_facade("facade_mesh")
    w, h, length, res, trunc = 96, 72, 2.0, 96, 0.06
    cams = ring_cameras(4, w, h)
    K = cams[0][0]
    rng = np.random.default_rng(6)
    depth = np.stack([np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16) for _, E in cams])
    color = rng.integers(0, 256, (len(cams), h, w, 3), dtype=np.uint8)
    vol = I.UniformTSDFVolume(length, res, trunc, I.TSDFVolumeColorType.RGB8)
    intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    for f, (_, E) in enumerate(cams):
        vol.integrate(G.RGBDImage.create_from_color_and_depth(G.Image(color[f]), G.Image(depth[f]), 1000.0, 100.0, False), intr, E)
    mesh = vol.extract_triangle_mesh()
    mesh.compute_vertex_normals()
    want = {"vertices": mesh.vertices.cpu(), "vertex_colors": mesh.vertex_colors.cpu(), "triangles": mesh.triangles.cpu(),
            "triangle_normals": mesh.triangle_normals.cpu(), "vertex_normals": mesh.vertex_normals.cpu()}
    with tempfile.TemporaryDirectory() as d:
        np.concatenate([[w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], len(cams), length, res, trunc]] +
                       [E.reshape(16) for _, E in cams]).astype(np.float32).tofile(os.path.join(d, "params.f32"))
        depth.tofile(os.path.join(d, "depth.u16"))
        color.tofile(os.path.join(d, "color.u8"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        for name, a in want.items():
            got = np.fromfile(os.path.join(d, "out_%s.%s" % (name, "i32" if name == "triangles" else "f32")), a.dtype).reshape(-1, 3)
            np.testing.assert_array_equal(got.view(np.uint32), np.ascontiguousarray(a).view(np.uint32), err_msg=name)
    assert len(want["triangles"]) > 100
