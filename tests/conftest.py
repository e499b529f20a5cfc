import os
import sys

import pytest

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(REPO, "arrow-rs_b200"))
sys.path.insert(0, os.path.dirname(__file__))
sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def gpu():
    """The product path: libarrow_cuda.so on cuda:0. No CPU fallback — fails loudly."""
    import acu
    ctx = acu.Context(0)
    yield ctx
    ctx.close()
