import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle_c():
    from oracle import oracle_c as oc
    oc.load()
    return oc


@pytest.fixture(scope="session")
def oracle_np():
    from oracle import bestfit_np
    return bestfit_np


@pytest.fixture(scope="session")
def egpu():
    import elastic_gpu_agent_b200 as e
    return e


@pytest.fixture()
def alloc(egpu):
    """A CUDA allocator context; GPU tests only.  Fails (does not skip) when the
    library or the device is missing: there is no CPU fallback to fall back to."""
    a = egpu.BestFitAllocator(0)
    yield a
    a.close()
