import os
import sys

import os

# several estimator contexts of one process wait for each other inside kernels (two-rank tests on one GPU): give every stream its own
# hardware queue so that a spinning wait kernel can never sit in front of the kernel it waits for
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle_py
    oracle_py.build()
    return oracle_py
