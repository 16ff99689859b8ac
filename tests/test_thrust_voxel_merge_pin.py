"""CPU: VoxelGrid's AddVoxels and operator+= as thrust itself computes them (tests/cpp/thrust_voxel_merge_pin.cpp, the
toolkit's thrust compiled for the CPP backend) equal the oracle's restatement (oracle/voxelgrid_ops.c), which the device
matches bit for bit.  This pins what DESIGN §4 item 17 mirrors: sort_by_key on lexicographic Vector3i keys is stable,
unique_by_key keeps the first entry of each run (the existing voxel), and reduce_by_key sums a run left to right in
that order before the division by the count.  Runs of two (the project's own unique grids) and runs of up to a dozen
(assigned keys that repeat) are both covered."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import voxelgrid_ops_py as V

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
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + inc,
                           "-DTHRUST_DEVICE_SYSTEM=THRUST_DEVICE_SYSTEM_CPP",
                           os.path.join(ROOT, "tests", "cpp", "thrust_voxel_merge_pin.cpp"), "-o", exe])
    yield exe, d
    shutil.rmtree(d, ignore_errors=True)


def run(pin, keys, cols):
    exe, d = pin
    src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(src, "wb") as f:
        np.int32(len(keys)).tofile(f)
        np.ascontiguousarray(keys, np.int32).tofile(f)
        np.ascontiguousarray(cols, np.float32).tofile(f)
    subprocess.check_call([exe, src, dst])
    raw = np.fromfile(dst, np.uint8)
    out, off = [], 0
    for _ in range(2):
        m = int(raw[off:off + 4].view(np.int32)[0])
        off += 4
        k = raw[off:off + 12 * m].view(np.int32).reshape(m, 3)
        off += 12 * m
        c = raw[off:off + 12 * m].view(np.float32).reshape(m, 3)
        off += 12 * m
        out.append((k, c))
    return out


@pytest.mark.parametrize("case", ["two_unique_grids", "repeated_keys", "one_key"])
def test_thrust_add_voxels_and_iadd_equal_the_oracle(pin, case):
    rng = np.random.default_rng(21)
    if case == "two_unique_grids":
        ka = np.unique(rng.integers(-8, 8, (3000, 3)), axis=0)
        kb = np.unique(rng.integers(-4, 12, (3000, 3)), axis=0)
    elif case == "repeated_keys":  # runs of up to a dozen entries, in any order
        ka, kb = rng.integers(0, 5, (700, 3)), rng.integers(0, 5, (600, 3))
    else:
        ka, kb = np.zeros((7, 3), int), np.zeros((5, 3), int)
    ka, kb = ka.astype(np.int32), kb.astype(np.int32)
    ca, cb = rng.random((len(ka), 3)).astype(np.float32), rng.random((len(kb), 3)).astype(np.float32)
    (k_add, c_add), (k_sum, c_sum) = run(pin, np.concatenate([ka, kb]), np.concatenate([ca, cb]))
    w_add, w_sum = V.merge(ka, ca, kb, cb, False), V.merge(ka, ca, kb, cb, True)
    np.testing.assert_array_equal(k_add, w_add[0])
    np.testing.assert_array_equal(c_add.view(np.uint32), w_add[1].view(np.uint32))
    np.testing.assert_array_equal(k_sum, w_sum[0])
    np.testing.assert_array_equal(c_sum.view(np.uint32), w_sum[1].view(np.uint32))
    assert len(k_sum) < len(ka) + len(kb)
