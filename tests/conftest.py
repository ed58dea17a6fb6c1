import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def cuda_dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from rainbow_iqn_apex_b200 import _lib
    _lib.require_device()
    return torch.device("cuda")
