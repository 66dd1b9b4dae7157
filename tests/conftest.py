import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a; select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """contract-math oracle (bit-identical arithmetic to the CUDA kernels)"""
    import _oracle
    _oracle.build_oracle()
    return _oracle.load(libm=False)


@pytest.fixture(scope="session")
def oracle_libm():
    """glibc-libm oracle (the arithmetic the Rust reference performs)"""
    import _oracle
    _oracle.build_oracle()
    return _oracle.load(libm=True)
