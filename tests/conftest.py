import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90)")


def golden_names():
    return sorted(os.path.basename(p)[4:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "cca_*.npz")))


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, f"cca_{name}.npz")))


@pytest.fixture(params=golden_names())
def golden(request):
    g = load_golden(request.param)
    g["name"] = request.param
    return g
