import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def ctx():
    """One tgpu_ctx on cuda:0 for the whole GPU session."""
    from trino_b200.operators import Context
    c = Context(0)
    yield c
    c.close()
