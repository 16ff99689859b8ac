"""cphb_scratch and cphb_arena, the owners of an entry point's device scratch and of a handle's device block
(cupoch_b200/csrc/cphb_internal.cuh): the types checked on the host against recording stubs of the allocator, and a
source check that no hand-written free list comes back."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from cupoch_b200.build import FLAGS, NVCC, SRC

# the only places that may call cphb_free_async or cudaFreeAsync: the owners themselves (None: the whole file), the
# allocator, and the storage that outlives a call -- the distance transform's grid, the occupancy grid, the neighbour table
FREE_ALLOWED = {
    "cphb_internal.cuh": None,
    "index.cu": {"cphb_free_async", "cphb_reserve_pool", "cphb_free"},
    "edt.cu": {"edt_alloc_grid", "cphb_dt_reconstruct", "cphb_dt_destroy"},
    "occgrid.cu": {"cphb_occgrid_create", "cphb_occgrid_destroy"},
    "search.cu": {"cphb_nbr_table_release"},
}
# a function definition starts in column 0: [extern "C"] [static] <type> <name>(
_DEF = re.compile(r'^(?:extern "C" )?[A-Za-z_][\w\s*]*?\b(\w+)\(')


def test_scratch_frees_every_buffer_once(tmp_path):
    if not os.access(NVCC, os.X_OK):
        pytest.skip("nvcc not found")
    exe = str(tmp_path / "scratch_check")
    subprocess.check_call([NVCC] + FLAGS + [os.path.join(ROOT, "tests", "cpp", "scratch_check.cu"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "scratch_check: ok" in r.stdout


def test_no_hand_written_free_lists():
    stray = []
    for name in sorted(os.listdir(SRC)):
        if not name.endswith((".cu", ".cuh")):
            continue
        allowed = FREE_ALLOWED.get(name, set())
        func = None
        with open(os.path.join(SRC, name)) as f:
            for no, line in enumerate(f, 1):
                m = _DEF.match(line)
                if m:
                    func = m.group(1)
                if ("cphb_free_async(" in line or "cudaFreeAsync(" in line) and allowed is not None and func not in allowed:
                    stray.append("%s:%d in %s" % (name, no, func))
    assert not stray, "device storage belongs to a cphb_scratch or a cphb_arena: " + ", ".join(stray)
