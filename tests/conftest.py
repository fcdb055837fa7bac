import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _native_build():
    from tepdist_b200 import build_native
    try:
        build_native.build_all()
    except Exception as e:  # pragma: no cover
        print("native build failed:", e)
    yield
