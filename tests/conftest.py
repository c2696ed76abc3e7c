"""pytest config: registers the `gpu` marker; builds the oracle (test infrastructure) on demand."""
import importlib
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
PKG_NAME = "llm-d-workload-variant-autoscaler_b200"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def pkg():
    """The product package (hyphenated directory name -> importlib)."""
    return importlib.import_module(PKG_NAME)


@pytest.fixture(scope="session")
def oracle():
    from tests import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def engine(pkg):
    """A live GPU context through the C-ABI; fails loudly when the CUDA library is missing."""
    eng = pkg.Engine(device=0)
    yield eng
    eng.close()
