import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (H100) device; run on the GPU box with -m gpu")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    def load(name):
        return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    return load
