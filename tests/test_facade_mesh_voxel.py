"""VoxelGrid::CreateFromTriangleMesh[WithinBounds] through the C++ facade (tests/cpp/facade_mesh_voxel.cpp): compiles and
links with plain g++ (CPU); on the GPU its known answers hold and both grids of a TSDF sphere mesh equal the Python
path's bit for bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_mesh_voxel_compiles_and_links():
    exe = build_facade("facade_mesh_voxel")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


@pytest.mark.gpu
def test_facade_mesh_voxel_matches_the_python_path():
    import cupoch_b200 as cph
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    G, I = cph.geometry, cph.integration
    exe = build_facade("facade_mesh_voxel")
    w, h = 96, 72
    vol = I.UniformTSDFVolume(2.0, 96, 0.06, I.TSDFVolumeColorType.NoColor)
    for K, E in ring_cameras(4, w, h):
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        im = G.RGBDImage.create_from_color_and_depth(G.Image(np.zeros((h, w, 3), np.uint8)), G.Image(d16), 1000.0, 100.0)
        vol.integrate(im, cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    mesh = vol.extract_triangle_mesh()
    v, t = mesh.vertices.cpu(), mesh.triangles.cpu()
    assert len(t) > 100
    vs, lo, hi = 0.03, (-0.5, -0.7, -0.1), (0.7, 0.4, 0.8)
    grids = {"within": G.VoxelGrid.create_from_triangle_mesh_within_bounds(mesh, vs, lo, hi),
             "own": G.VoxelGrid.create_from_triangle_mesh(mesh, vs)}
    with tempfile.TemporaryDirectory() as d:
        v.astype(np.float32).tofile(os.path.join(d, "mesh.f32"))
        t.astype(np.int32).tofile(os.path.join(d, "mesh.i32"))
        np.array((vs,) + lo + hi, np.float32).tofile(os.path.join(d, "bounds.f32"))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        for name, g in grids.items():
            keys, cols = g.get_voxels()
            assert len(keys) > 100
            got_k = np.fromfile(os.path.join(d, "out_%s_keys.i32" % name), np.int32).reshape(-1, 3)
            got_c = np.fromfile(os.path.join(d, "out_%s_colors.f32" % name), np.float32).reshape(-1, 3)
            geo = np.fromfile(os.path.join(d, "out_%s_geometry.f32" % name), np.float32)
            np.testing.assert_array_equal(got_k, keys, err_msg=name)
            np.testing.assert_array_equal(got_c.view(np.uint32), cols.view(np.uint32), err_msg=name)
            np.testing.assert_array_equal(geo.view(np.uint32), np.append(np.float32(g.voxel_size), g.origin).view(np.uint32))
