import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    oracle_lib.build()
    return oracle_lib


@pytest.fixture(scope="session")
def z():
    """the product package, initialised on cuda:0; GPU tests fail loudly if the native library cannot run"""
    import sharpziplib_b200
    sharpziplib_b200.init(0)
    return sharpziplib_b200
