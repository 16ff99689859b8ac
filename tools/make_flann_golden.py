#!/usr/bin/env python3
"""Generate tests/golden/flann_ref.npz: what the reference's own search engine -- the FLANN CUDA kd-tree cupoch
vendors, built into oracle/_ref/libflann_ref.so by oracle/ref_flann/Makefile -- returns on the inputs of
tests/test_gpu_flann_ref.py.

Needs a GPU and oracle/_ref/libflann_ref.so.  FLANN runs on every query of each case, exactly as the test used to
call it; the file keeps a fixed, seeded sample of the rows (all rows of the small lattice case) so that it stays
small:  <case>_rows (query indices, ascending), <case>_idx and <case>_d2 ([rows][k], FLANN's int32 / float32).

    python tools/make_flann_golden.py [OUT.npz]
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cupoch_b200.testing import datagen  # noqa: E402

SO = os.path.join(ROOT, "oracle", "_ref", "libflann_ref.so")
OUT = os.path.join(ROOT, "tests", "golden", "flann_ref.npz")


def lattice_case():
    g = np.stack(np.meshgrid(*[np.arange(12, dtype=np.float32)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.25
    tgt = np.concatenate([g, g[::3], g[::7]]).astype(np.float32)
    tgt = tgt[np.random.default_rng(3).permutation(len(tgt))]
    qry = np.concatenate([g + 0.125, g]).astype(np.float32)
    return tgt, qry


def cases():
    """(name, target, queries, kind, radius, k, sampled rows); kept in step with tests/test_gpu_flann_ref.py"""
    def rows(n, m, seed):
        return np.sort(np.random.default_rng(seed).choice(n, size=min(m, n), replace=False)).astype(np.int32)
    u_tgt = datagen.uniform_cube(200_000, 101)
    u_qry = datagen.uniform_cube(100_000, 202, lo=(-0.05, -0.05, -0.05), hi=(1.05, 1.05, 1.05))
    yield "uniform_r0.02", u_tgt, u_qry, "radius", 0.02, 1, rows(len(u_qry), 2048, 1)
    yield "uniform_r0.3", u_tgt, u_qry, "radius", 0.3, 1, rows(len(u_qry), 2048, 2)
    tgt, _ = datagen.surface(1_000_000, 11)
    src = datagen.make_source(tgt, datagen.gt_transform(), 13, 14, 5e-4)
    yield "config2", tgt, src, "radius", 0.02, 1, rows(len(src), 2048, 3)
    tgt, qry = lattice_case()
    yield "lattice", tgt, qry, "radius", 0.5, 1, np.arange(len(qry), dtype=np.int32)
    tgt, qry = datagen.uniform_cube(20_000, 5), datagen.uniform_cube(5_000, 6)
    for k, r in ((4, 0.05), (15, 0.08), (30, 0.1)):
        yield "radius_k%d" % k, tgt, qry, "radius", r, k, rows(len(qry), 128, 4)
    tgt, qry = datagen.uniform_cube(50_000, 7), datagen.uniform_cube(5_000, 8)
    yield "knn30", tgt, qry, "knn", 0.0, 30, rows(len(qry), 128, 5)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    L = C.CDLL(SO)
    L.fref_build.restype = C.c_void_p
    L.fref_build.argtypes = [C.c_void_p, C.c_int]
    L.fref_free.argtypes = [C.c_void_p]
    L.fref_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.fref_radius.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    data = {}
    for name, tgt, qry, kind, r, k, rows in cases():
        tgt, qry = np.ascontiguousarray(tgt, np.float32), np.ascontiguousarray(qry, np.float32)
        h = L.fref_build(tgt.ctypes.data, len(tgt))
        assert h, "the reference's FLANN index failed to build"
        idx = np.empty((len(qry), k), np.int32)
        d2 = np.empty((len(qry), k), np.float32)
        if kind == "knn":
            rc = L.fref_knn(h, qry.ctypes.data, len(qry), k, idx.ctypes.data, d2.ctypes.data)
        else:
            rc = L.fref_radius(h, qry.ctypes.data, len(qry), C.c_float(r), k, idx.ctypes.data, d2.ctypes.data)
        L.fref_free(h)
        assert rc == 0, name
        data[name + "_rows"], data[name + "_idx"], data[name + "_d2"] = rows, idx[rows], d2[rows]
        print(name, len(qry), "queries,", len(rows), "kept")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **data)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
