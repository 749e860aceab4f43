import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")


@pytest.fixture(scope="session")
def oracle():
    """CPU restatement of the reference (oracle/): the checker, never the thing under test."""
    from oracle import oracle as O
    O.lib()
    return O


@pytest.fixture(scope="session")
def ctx():
    from loam_livox_b200.registration import Context
    c = Context(0, max_scan_points=400000, max_features=400000)
    yield c
    c.close()
