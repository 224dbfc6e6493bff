import os
import sys

import pytest

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (REPO, os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(REPO, "tests", "golden")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Make sure the in-tree CUDA library exists (nvcc cross-compiles without a GPU)."""
    from triforce_b200 import build
    build.build(verbose=False)
