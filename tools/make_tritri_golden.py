#!/usr/bin/env python3
"""Write tests/golden/tritri_ref.npz: the reference's own triangle/triangle answers (oracle/_ref/libtritri_ref.so, built by
oracle/ref_tritri/Makefile from a cupoch checkout's opttritri.h) on a seeded set of raw pairs, so that the CPU oracle and
the device predicate can be checked against the reference's code where the reference is absent.

    python tools/make_tritri_golden.py REF=<cupoch checkout>

Pair families (`kind`): 0 random, 1 touching at a vertex, 2 touching along an edge, 3 coplanar overlapping, 4 coplanar
disjoint, 5 parallel planes, 6 |du0| within a few ULPs of the published EPSILON (1e-6), 7 nearly degenerate first
triangle, 8 nearly degenerate second triangle.  Arrays: p, q [n, 3, 3] float32, hit [n] uint8, kind [n] uint8."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def normalise(p, q):
    """intersection_test.inl's mean / sigma normalisation in float32, Eigen's evaluation order"""
    six = np.concatenate([p, q]).astype(F)
    mu = ((((((six[0] + six[1]) + six[2]) + six[3]) + six[4]) + six[5]) / F(6)).astype(F)
    d = (six - mu).astype(F)
    sq = d * d
    s = (((((sq[0] + sq[1]) + sq[2]) + sq[3]) + sq[4]) + sq[5]).astype(F)
    sg = (np.sqrt((s / F(5)).astype(F)).astype(F) + F(1e-12)).astype(F)
    m = (d / sg).astype(F)
    return m[:3], m[3:]


def du0(p, q):
    """NoDivTriTriIsect's du0 = DOT(N1, U0) + d1 on the normalised pair, float32 in the published order"""
    V, U = normalise(p, q)
    e1, e2 = (V[1] - V[0]).astype(F), (V[2] - V[0]).astype(F)
    n = np.array([e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]], F)
    d1 = F(-((n[0] * V[0][0] + n[1] * V[0][1]) + n[2] * V[0][2]))
    return F(((n[0] * U[0][0] + n[1] * U[0][1]) + n[2] * U[0][2]) + d1)


def families(rng, per):
    out = []
    tri = lambda: rng.uniform(-1, 1, (3, 3)).astype(F)
    for _ in range(per):  # 0 random (half of them overlapping in the box)
        out.append((0, tri(), tri() * F(rng.choice([0.5, 1.0]))))
    for _ in range(per):  # 1 vertex touch: q starts at a vertex of p
        p, q = tri(), tri()
        q = (q - q[0] + p[rng.integers(3)]).astype(F)
        out.append((1, p, q))
    for _ in range(per):  # 2 edge touch: q's vertex on p's edge midpoint
        p, q = tri(), tri()
        a = rng.integers(3)
        q = (q - q[0] + (p[a] + p[(a + 1) % 3]) * F(0.5)).astype(F)
        out.append((2, p, q))
    for _ in range(per):  # 3 / 4 coplanar, overlapping or shifted apart in the plane
        p, q = tri(), tri()
        p[:, 2] = q[:, 2] = F(rng.uniform(-1, 1))
        out.append((3, p, (q * F(0.5) + p.mean(0) * F(0.5)).astype(F)))
        out.append((4, p, (q + F(5)).astype(F) * np.array([1, 1, 0], F) + p[:, 2:3].mean() * np.array([0, 0, 1], F)))
    for _ in range(per):  # 5 parallel planes
        p = tri()
        out.append((5, p, (p[[1, 2, 0]] + np.array([0.1, -0.1, rng.uniform(0.001, 0.5)], F)).astype(F)))
    for _ in range(per):  # 6 |du0| near EPSILON: U0 moved off p's plane until |du0| crosses 1e-6, then +-4 ULPs around it
        p, q = tri(), tri()
        nrm = np.cross(p[1] - p[0], p[2] - p[0]).astype(np.float64)
        nrm /= np.linalg.norm(nrm)
        base = q.copy()
        base[0] = (p.mean(0) + (q[0] - p.mean(0)) - nrm * np.dot(q[0] - p.mean(0), nrm)).astype(F)
        lo, hi = 0.0, 1e-3
        for _ in range(80):
            mid = 0.5 * (lo + hi)
            qq = base.copy()
            qq[0] = (base[0] + nrm * mid).astype(F)
            if abs(float(du0(p, qq))) < 1e-6:
                lo = mid
            else:
                hi = mid
        for k in range(-4, 5):
            qq = base.copy()
            qq[0] = (base[0] + nrm * hi).astype(F)
            qq[0, 2] = np.nextafter(qq[0, 2], F(np.inf) if k > 0 else F(-np.inf)) if k else qq[0, 2]
            for _ in range(abs(k) - 1):
                qq[0, 2] = np.nextafter(qq[0, 2], F(np.inf) if k > 0 else F(-np.inf))
            out.append((6, p, qq.astype(F)))
    for _ in range(per):  # 7 / 8 nearly degenerate: three almost collinear points
        a, d = rng.uniform(-1, 1, 3), rng.normal(size=3)
        s = (np.array([a, a + d, a + d * rng.uniform(0, 1) + rng.normal(size=3) * 10 ** rng.uniform(-7, -3)])).astype(F)
        out.append((7, s, tri()))
        out.append((8, tri(), s))
    return out


def main():
    ref = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("REF=")]
    if not ref:
        sys.exit("usage: make_tritri_golden.py REF=<cupoch checkout>")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle", "ref_tritri"), "REF=" + ref[0]])
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libtritri_ref.so"))
    rows = families(np.random.default_rng(20261019), 400)
    kind = np.array([r[0] for r in rows], np.uint8)
    p = np.ascontiguousarray(np.stack([r[1] for r in rows]), F)
    q = np.ascontiguousarray(np.stack([r[2] for r in rows]), F)
    hit = np.zeros(len(rows), np.uint8)
    lib.ref_tritri_many(p.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), C.c_longlong(len(rows)), hit.ctypes.data_as(C.c_void_p))
    out = os.path.join(ROOT, "tests", "golden", "tritri_ref.npz")
    np.savez_compressed(out, p=p, q=q, hit=hit, kind=kind)
    print(out, len(rows), "pairs,", int(hit.sum()), "hits; per kind", np.bincount(kind).tolist(),
          "hits per kind", np.bincount(kind, weights=hit).astype(int).tolist())


if __name__ == "__main__":
    main()
