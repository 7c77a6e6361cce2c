import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run on a GPU machine with `-m gpu`)")


@pytest.fixture(scope="session")
def oracle():
    """ctypes handle on the CPU oracle (test infrastructure only)."""
    import oracle_lib
    return oracle_lib.load_oracle()


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference templates compiled into oracle/_ref (None if it was never built)."""
    import oracle_lib
    return oracle_lib.load_ref()


@pytest.fixture(scope="session")
def fecc():
    """The product library, initialised on cuda:0 (GPU tests only)."""
    from fastecc_b200 import build as _b
    _b.build()
    import fastecc_b200
    fastecc_b200.init(0)
    return fastecc_b200
