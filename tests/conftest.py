import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    def load(name):
        return dict(np.load(os.path.join(GOLDEN, name)))
    return load


@pytest.fixture(scope="session")
def po():
    from oracle import pyoracle
    pyoracle.lib()
    return pyoracle


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from orientedreppoints_b200 import _lib
    _lib.lib()   # must load - no fallback
    return torch.device("cuda", 0)
