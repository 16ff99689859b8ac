"""TriangleMesh cleanup, GetSelfIntersectingTriangles and + / += through the C++ facade (tests/cpp/facade_mesh_clean.cpp):
compiles and links with plain g++ (CPU); on the GPU its known answers hold and every result equals the Python path's
bit for bit."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_facade_cpp import build_facade


def test_facade_mesh_clean_compiles_and_links():
    exe = build_facade("facade_mesh_clean")
    out = subprocess.run(["ldd", exe], capture_output=True, text=True).stdout
    assert "libcupoch_b200.so" in out and "not found" not in out


def _mesh(seed, nv, nt, q=3):
    rng = np.random.default_rng(seed)
    v = (rng.integers(-q, q + 1, (nv, 3)) / np.float32(q)).astype(np.float32)
    v[3] = (np.nan, 0, 0)
    t = rng.integers(0, nv, (nt, 3)).astype(np.int32)
    t[::7, 1] = t[::7, 0]
    return v, t, rng


@pytest.mark.gpu
def test_facade_mesh_clean_matches_the_python_path():
    import cupoch_b200 as cph
    G = cph.geometry
    exe = build_facade("facade_mesh_clean")
    va, ta, rng = _mesh(1, 1500, 2500)
    na, ca, tna = (rng.normal(size=(1500, 3)).astype(np.float32), rng.random((1500, 3)).astype(np.float32),
                   rng.normal(size=(2500, 3)).astype(np.float32))
    c = rng.uniform(0, 1, (800, 1, 3))
    vb = (c + rng.normal(size=(800, 3, 3)) * 0.05).reshape(-1, 3).astype(np.float32)
    tb = np.arange(2400, dtype=np.int32).reshape(-1, 3)

    def py_a():
        m = G.TriangleMesh(va, ta)
        m.vertex_normals, m.vertex_colors, m.triangle_normals = na, ca, tna
        return m.compute_edge_list()

    b = G.TriangleMesh(vb, tb)
    a = py_a()
    want = {"sum": py_a() + b}
    acc = py_a()
    acc += b
    want["acc"] = acc
    for name, op in (("dv", "remove_duplicated_vertices"), ("dt", "remove_duplicated_triangles"),
                     ("dg", "remove_degenerate_triangles"), ("ur", "remove_unreferenced_vertices")):
        getattr(a, op)()
        want[name] = {"v": a.vertices.cpu(), "t": a.triangles.cpu(), "n": a.vertex_normals.cpu(), "c": a.vertex_colors.cpu(),
                      "tn": a.triangle_normals.cpu(), "e": a.edge_list.cpu()}
    self_b = b.get_self_intersecting_triangles().cpu()
    assert len(self_b) > 0
    with tempfile.TemporaryDirectory() as d:
        for name, arr in (("a.f32", va), ("a.i32", ta), ("a_n.f32", na), ("a_c.f32", ca), ("a_tn.f32", tna), ("b.f32", vb), ("b.i32", tb)):
            arr.tofile(os.path.join(d, name))
        r = subprocess.run([exe, d], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr

        def got(name, part, dtype):
            return np.fromfile(os.path.join(d, "out_%s_%s.%s" % (name, part, "i32" if dtype == np.int32 else "f32")), dtype)

        for name in ("sum", "acc"):
            m = want[name]
            want[name] = {"v": m.vertices.cpu(), "t": m.triangles.cpu(), "n": np.zeros((0, 3), np.float32),
                          "c": np.zeros((0, 3), np.float32), "tn": np.zeros((0, 3), np.float32), "e": m.edge_list.cpu()}
            assert not m.has_vertex_normals() and not m.has_vertex_colors() and not m.has_triangle_normals()
        for name, w in want.items():
            for part, arr in w.items():
                dt = np.int32 if part in ("t", "e") else np.float32
                g = got(name, part, dt)
                ref = np.ascontiguousarray(arr, dt).reshape(-1)
                assert g.shape == ref.shape, (name, part)
                assert np.array_equal(g.view(np.uint32) if dt == np.float32 else g, ref.view(np.uint32) if dt == np.float32 else ref), (name, part)
        np.testing.assert_array_equal(np.fromfile(os.path.join(d, "out_self_b.i32"), np.int32).reshape(-1, 2), self_b)
