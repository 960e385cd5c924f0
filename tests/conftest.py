import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA sm_90 (H100) device; run with -m gpu")


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree CUDA library; built on demand (cross-compiles without a GPU)."""
    from pixie_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


@pytest.fixture(scope="session")
def cuda_dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return "cuda:0"
