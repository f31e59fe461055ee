import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


@pytest.fixture(scope="session")
def golden_doremi():
    return load_golden("doremi.npz")


@pytest.fixture(scope="session")
def golden_synth():
    return load_golden("synthetic.npz")


@pytest.fixture(scope="session")
def golden_edges():
    return load_golden("edges.npz")


@pytest.fixture(scope="session")
def golden_pytests():
    return load_golden("pytests.npz")
