import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with -m gpu)")


def _oracle_kinds():
    from oracle import pyoracle
    kinds = [k for k in ("reference", "port") if pyoracle.available(k)]
    return kinds


@pytest.fixture(scope="session")
def oracle_kinds():
    return _oracle_kinds()


def pytest_generate_tests(metafunc):
    if "ora_kind" in metafunc.fixturenames:
        kinds = _oracle_kinds()
        metafunc.parametrize("ora_kind", kinds if kinds else ["none"])
