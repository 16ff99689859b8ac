"""ctypes loader for the ExtractTriangleMesh and mesh-normal restatement (oracle/tsdf_mesh.c).

TEST INFRASTRUCTURE ONLY, like oracle_py: imported by tests/ and tools/, never by the product package cupoch_b200/.  The
library is built by oracle.build("tsdf_mesh").  The volume is a tsdf_py.Volume (its host planes are read as they are).
"""
import ctypes as C

import numpy as np

from . import build as _build, load, ptr as _p

INT32_MAX = 2 ** 31 - 1


def build(force=False):
    return _build("tsdf_mesh", force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load("tsdf_mesh")
        _lib.orc_tsdf_mesh_extract.restype = C.c_longlong
        for f in ("orc_mesh_triangle_normals", "orc_mesh_vertex_normals", "orc_mc_tables"):
            getattr(_lib, f).restype = C.c_int
    return _lib


def tables():
    """the compiled tables -> (edge table [256] uint16, triangle counts [256] uint8, triangle table [256, 3 * max] int8)"""
    e, c, t = np.empty(256, np.uint16), np.empty(256, np.uint8), np.empty(256 * 3 * 16, np.int8)
    m = lib().orc_mc_tables(_p(e), _p(c), _p(t))
    return e, c, t[:256 * 3 * m].reshape(256, 3 * m)


def extract_triangle_mesh(vol, max_vertices=INT32_MAX):
    """ExtractTriangleMesh of a tsdf_py.Volume -> (vertices [n, 3] float32, vertex colours [n, 3] float32 or None for
    NoColor, triangles [m, 3] int32); ValueError when the vertex count exceeds max_vertices"""
    L = lib()
    args = (_p(vol.tw), _p(vol.col), C.c_float(vol.length), C.c_int(vol.res), C.c_int(vol.ct), _p(vol.origin))
    nt = C.c_longlong(0)
    nv = L.orc_tsdf_mesh_extract(*args, None, None, None, C.c_longlong(0), C.c_longlong(0), C.c_longlong(max_vertices), C.byref(nt))
    if nv < 0:
        raise ValueError("the mesh has more than %d vertices" % max_vertices)
    m = nt.value
    v, c, t = np.empty((max(nv, 1), 3), np.float32), np.empty((max(nv, 1), 3), np.float32), np.empty((max(m, 1), 3), np.int32)
    L.orc_tsdf_mesh_extract(*args, _p(v), _p(c), _p(t), C.c_longlong(nv), C.c_longlong(m), C.c_longlong(max_vertices), C.byref(nt))
    return v[:nv], (c[:nv] if vol.ct != 0 else None), t[:m]


def triangle_normals(vertices, triangles, normalized=True):
    v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
    t = np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
    out = np.empty((max(len(t), 1), 3), np.float32)
    if lib().orc_mesh_triangle_normals(_p(v), C.c_longlong(len(v)), _p(t), C.c_longlong(len(t)), C.c_int(int(normalized)), _p(out)):
        raise ValueError("a triangle's vertex index is outside [0, n_vertices)")
    return out[:len(t)]


def vertex_normals(n_vertices, triangles, tri_normals, normalized=True):
    t = np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
    tn = np.ascontiguousarray(tri_normals, np.float32).reshape(-1, 3)
    out = np.empty((max(n_vertices, 1), 3), np.float32)
    if lib().orc_mesh_vertex_normals(_p(t), C.c_longlong(len(t)), _p(tn), C.c_longlong(n_vertices), C.c_int(int(normalized)), _p(out)):
        raise ValueError("a triangle's vertex index is outside [0, n_vertices)")
    return out[:n_vertices]


def compute_vertex_normals(vertices, triangles, tri_normals=None, normalized=True):
    """TriangleMesh::ComputeVertexNormals: the unnormalised triangle normals first when there are none -> (vertex normals,
    the triangle normals the mesh then holds)"""
    if tri_normals is None:
        tri_normals = triangle_normals(vertices, triangles, False)
    return vertex_normals(len(vertices), triangles, tri_normals, normalized), tri_normals
