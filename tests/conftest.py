import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture
def reference(oracle, request):
    """The reference's own code, replayed from tests/golden (see tests/ref_golden.py)."""
    from ref_golden import Reference
    r = Reference(request.node.name, oracle)
    yield r
    r.close()
