"""CPU: TriangleMesh::RemoveDuplicatedVertices and RemoveDuplicatedTriangles as thrust itself computes them
(tests/cpp/thrust_mesh_clean_pin.cpp, the toolkit's thrust compiled for the CPP backend, with the reference's call
sequence and helper.h's operator<) equal the oracle's restatement (oracle/mesh_clean.c), which the device matches bit
for bit.  This pins the survivor rules DESIGN §4 item 26 states: sort_by_key on Vector3f and Vector3i keys keeps equal
keys in their original order, so unique_by_key keeps the vertex normal of the lowest original index and the triangle
normal of the first of each run; reduce_by_key / exclusive_scan give the remap.  Inputs have runs of up to dozens of
equal keys, and -0 / +0 (no NaN: the reference's comparator is not a strict weak order with it)."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import mesh_clean_py as MC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _thrust_include():
    for d in (os.environ.get("CUDA_HOME", ""), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "include", "thrust", "sort.h")):
            return os.path.join(d, "include")
    return None


@pytest.fixture(scope="module")
def pin():
    inc = _thrust_include()
    if inc is None or shutil.which("g++") is None:
        pytest.skip("needs g++ and the CUDA toolkit's thrust headers")
    d = tempfile.mkdtemp()
    exe = os.path.join(d, "pin")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + inc, "-DTHRUST_DEVICE_SYSTEM=THRUST_DEVICE_SYSTEM_CPP",
                           os.path.join(ROOT, "tests", "cpp", "thrust_mesh_clean_pin.cpp"), "-o", exe])
    yield exe, d
    shutil.rmtree(d, ignore_errors=True)


def run(pin, v, n, t, tn):
    exe, d = pin
    src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(src, "wb") as f:
        np.int32(len(v)).tofile(f)
        v.tofile(f)
        n.tofile(f)
        np.int32(len(t)).tofile(f)
        t.tofile(f)
        tn.tofile(f)
    subprocess.check_call([exe, src, dst])
    raw = np.fromfile(dst, np.uint8)
    k = int(raw[:4].view(np.int32)[0])
    o = 4
    ov = raw[o:o + 12 * k].view(np.float32).reshape(k, 3)
    o += 12 * k
    on = raw[o:o + 12 * k].view(np.float32).reshape(k, 3)
    o += 12 * k
    ot = raw[o:o + 12 * len(t)].view(np.int32).reshape(-1, 3)
    o += 12 * len(t)
    k2 = int(raw[o:o + 4].view(np.int32)[0])
    o += 4
    t2 = raw[o:o + 12 * k2].view(np.int32).reshape(k2, 3)
    o += 12 * k2
    tn2 = raw[o:o + 12 * k2].view(np.float32).reshape(k2, 3)
    return ov, on, ot, t2, tn2


@pytest.mark.parametrize("q,nv,nt", [(2, 3000, 4000), (1, 800, 3000), (6, 20000, 20000)])
def test_thrust_remove_duplicated_equals_the_oracle(pin, q, nv, nt):
    rng = np.random.default_rng(q * 31 + nv)
    v = (rng.integers(-q, q + 1, (nv, 3)) / np.float32(max(q, 1))).astype(np.float32)
    v[rng.random(nv) < 0.1] *= np.float32(-1)  # -0 among +0
    n = rng.normal(size=(nv, 3)).astype(np.float32)
    t = rng.integers(0, min(nv, 12), (nt, 3)).astype(np.int32)  # few distinct indices: long runs of equal triangles
    tn = rng.normal(size=(nt, 3)).astype(np.float32)
    ov, on, ot, t2, tn2 = run(pin, v, n, t, tn)
    wv, wt, wn, _ = MC.remove_duplicated_vertices(v, t, n)
    assert len(wv) < nv // 2
    np.testing.assert_array_equal(ov.view(np.uint32), wv.view(np.uint32))
    np.testing.assert_array_equal(on.view(np.uint32), wn.view(np.uint32))
    np.testing.assert_array_equal(ot, wt)
    wt2, wtn2 = MC.remove_duplicated_triangles(t, nv, tn)
    assert len(wt2) < nt // 2
    np.testing.assert_array_equal(t2, wt2)
    np.testing.assert_array_equal(tn2.view(np.uint32), wtn2.view(np.uint32))
