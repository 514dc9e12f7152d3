import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def lib_path():
    """Builds libb200w.so if it is not there yet (nvcc cross-compiles without a GPU)."""
    from runbooks_b200 import build

    return build.build()


@pytest.fixture(scope="session")
def engine(lib_path):
    from runbooks_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()
