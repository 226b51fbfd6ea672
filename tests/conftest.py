import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "reference_golden.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def orc():
    from oracle import oracle
    oracle.build()
    return oracle
