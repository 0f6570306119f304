import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_masks.npz"))


@pytest.fixture(scope="session")
def maps():
    import cases
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = cases.MAPS[name]()
        return cache[name]
    return get


@pytest.fixture(scope="session")
def port_lib():
    from oracle import orc
    orc.build("port")
    return orc
