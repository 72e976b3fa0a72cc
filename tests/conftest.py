import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def pkg():
    return importlib.import_module("batch-scheduler_b200")


@pytest.fixture(scope="session")
def snapshot_mod():
    return importlib.import_module("batch-scheduler_b200.snapshot")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    return o
