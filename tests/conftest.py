import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """tests/golden/<name>.npz -> dict of torch tensors / python scalars."""
    out = {}
    with np.load(os.path.join(GOLDEN, name + ".npz")) as data:
        for key in data.files:
            arr = data[key]
            if arr.ndim == 0:
                out[key] = arr.item()
            else:
                t = torch.from_numpy(arr.copy())
                out[key] = t.float() if t.dtype == torch.float16 else t
    return out


@pytest.fixture
def golden():
    return load_golden
