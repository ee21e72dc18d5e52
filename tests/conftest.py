import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def _cuda_device_present() -> bool:
    try:
        import ctypes

        cu = ctypes.CDLL("libcuda.so.1")
        n = ctypes.c_int(0)
        return cu.cuInit(0) == 0 and cu.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return False


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests are the parity tests proper; on a box without a CUDA device they are skipped, not errored
    (the product itself still fails loudly: bgs_context_create returns BGS_ECUDA, there is no CPU path)."""
    if _cuda_device_present():
        return
    skip = pytest.mark.skip(reason="no CUDA device on this machine (run with -m gpu on an H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O

    O.load()
    return O
