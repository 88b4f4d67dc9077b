"""pytest configuration.

Two builds of the SAME native sources are exercised:
  * `-m gpu`      : zeekstd_b200/libzeekstd_b200.so (nvcc, sm_90a) on a real H100 -- the parity tests proper;
  * `-m "not gpu"`: tests/emul/_build/libzeekstd_b200_emul.so, the device code interpreted on the CPU by
                    tests/emul/cuda_emul.h (test infrastructure only) -- host logic + kernel logic on tiny inputs.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real CUDA device (run on an H100)")


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def emul_lib():
    from zeekstd_b200 import _native
    from zeekstd_b200.build import build_emul
    return _native.load(build_emul())


@pytest.fixture(scope="session")
def gpu_lib():
    from zeekstd_b200 import _native
    return _native.load(_native.PRODUCT_SO)
