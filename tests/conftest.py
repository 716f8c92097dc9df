import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine")


@pytest.fixture(scope="session")
def built_lib():
    """Path of the in-tree CUDA library (built on demand with nvcc; cross-compiles without a GPU)."""
    from turboprune_b200 import build
    return build.build()
