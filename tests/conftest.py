import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _gpu_usable():
    """the CUDA library is built and sees a device (no torch involved)"""
    try:
        from cupoch_b200 import _lib
        return _lib.lib().cphb_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a usable device must skip, not fail 50 tests and abort the C++ facade test
    if not any("gpu" in it.keywords for it in items):
        return
    if _gpu_usable():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device and the built libcupoch_b200.so")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "reference_vectors.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def orc():
    from oracle import oracle_py
    oracle_py.build()
    return oracle_py


def lexsort_rows(a):
    a = np.asarray(a)
    return a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))]
