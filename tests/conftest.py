import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """The C-ABI library must exist for both tiers (CPU tests only load it)."""
    from neuralmonkey_b200 import build
    build.build()
