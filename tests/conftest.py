import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def has_gpu():
    try:
        from tandem_b200._lib import lib
        return lib().tdm_device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def golden_small():
    return np.load(os.path.join(ROOT, "tests", "golden", "sample_512x320.npz"))


@pytest.fixture(scope="session")
def golden_full():
    return np.load(os.path.join(ROOT, "tests", "golden", "sample_640x480.npz"))


def pytest_collection_modifyitems(config, items):
    if has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
