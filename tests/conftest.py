import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100 with -m gpu)")


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)


@pytest.fixture(scope="session")
def golden():
    return load_golden


def sort_rows(a):
    """Rows of a 2-D array in lexicographic order (for set-level comparisons)."""
    a = np.asarray(a)
    if a.ndim == 1:
        return np.sort(a)
    return a[np.lexsort(a.T[::-1])]
