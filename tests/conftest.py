import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def engine_lib():
    """libb200tsdf.so, built in-tree; GPU tests fail loudly if it cannot be built or loaded."""
    from cpu_tsdf_b200.build import build_library
    return build_library()


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import oracle_py
    oracle_py.build()
    return oracle_py.load("port")
