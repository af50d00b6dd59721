import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    import oracle as o
    return o


@pytest.fixture(scope="session")
def ref(oracle):
    if oracle.ref is None:
        pytest.skip("oracle/_ref/liboracle_ref.so not built (no reference sources here)")
    return oracle.ref
