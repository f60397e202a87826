import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu where one is visible)")


@pytest.fixture(scope="session")
def engine_lib():
    """The CUDA library, built in-tree.  GPU tests must fail (not skip) if it cannot be loaded."""
    from hyphy_b200 import build, engine
    build.build()
    return engine.load_library()
