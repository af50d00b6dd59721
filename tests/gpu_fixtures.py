"""The fixtures the GPU test modules share.  A module imports them by name (`from gpu_fixtures import capi, engine`);
being module-scoped, each importing module still gets its own engine, closed after its last test."""
import pytest


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def capi():
    import gnss_sdr_b200.capi as c
    return c


@pytest.fixture(scope="module")
def engine(capi):
    e = capi.Engine(0)
    yield e
    e.close()
