import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _cuda_device_present():
    """True when the product library can create a context (a CUDA device is visible)."""
    try:
        from okvis_b200 import capi
        c = capi.Context(0, 1)
        c.close()
        return True
    except Exception as e:      # only OKB_ERR_NO_DEVICE (-5) means "CPU-only machine"; anything else (e.g. the
        return getattr(e, "code", None) != -5      # library is not built) must make the gpu tests run and fail loudly


def pytest_collection_modifyitems(config, items):
    """gpu-marked tests are skipped (not errored) on machines without a CUDA device; tests/test_abi.py keeps the
    dedicated check that the product fails loudly there."""
    gpu_items = [it for it in items if it.get_closest_marker("gpu")]
    if not gpu_items or _cuda_device_present():
        return
    skip = pytest.mark.skip(reason="no CUDA device (run with -m gpu on an H100)")
    for it in gpu_items:
        it.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Built on demand with g++."""
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="session")
def okb():
    """The product library through its C-ABI wrapper; fails loudly when it is not built."""
    from okvis_b200 import capi
    return capi
