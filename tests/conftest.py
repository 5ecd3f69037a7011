import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as orc
    orc.lib()
    return orc


@pytest.fixture(scope="session")
def gpu():
    """the product library (libsr_gpu.so) + one context on cuda:0"""
    from starrocks_b200 import gpu as g
    g.lib()
    return g


@pytest.fixture()
def ctx(gpu):
    c = gpu.Context(0)
    yield c
    c.close()
