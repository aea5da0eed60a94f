import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine with one)")


@pytest.fixture(scope="session")
def cuda_lib():
    """The in-tree CUDA library; GPU tests must go through it (no fallback)."""
    import torch
    assert torch.cuda.is_available(), "gpu-marked test running without a GPU"
    from buffalo_b200 import _cabi
    return _cabi.lib()
