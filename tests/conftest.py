import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def pkg():
    """The product package (its directory name is not a Python identifier, hence importlib)."""
    return importlib.import_module("end-to-end-asr-pytorch_b200")


def load_golden(name):
    from oracle import golden_io
    return golden_io.load(os.path.join(GOLDEN, name))


def rel_err(a, b, floor=1e-3):
    """max |a-b| / max(|b|, floor) - the tolerance form of SURVEY.md 8(c)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), floor))) if a.size else 0.0


def scaled_err(a, b):
    """max |a-b| / max |b|: error relative to the tensor's scale (for gradients with near-zero elements)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), 1e-30)) if a.size else 0.0
