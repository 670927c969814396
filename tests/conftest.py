import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session", autouse=True)
def _built_extension():
    """Make sure the in-tree extension exists (nvcc cross-compiles without a GPU)."""
    from centernet_b200.build import build
    build()
