import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) CUDA device; select with -m gpu")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    o.lib()
    return o
