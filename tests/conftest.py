import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_outputs.npz"))


def rel_errors(a, ref):
    """(max|a-ref|/max|ref|, ||a-ref||_2/||ref||_2) -- the two parity metrics of SURVEY 8(d)."""
    a = np.asarray(a, np.float64)
    ref = np.asarray(ref, np.float64)
    d = a - ref
    m = float(np.abs(d).max() / max(np.abs(ref).max(), 1e-30))
    l2 = float(np.sqrt((d ** 2).sum()) / max(np.sqrt((ref ** 2).sum()), 1e-30))
    return m, l2
