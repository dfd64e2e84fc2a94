import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_cuda = torch.cuda.is_available()
    except Exception:
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session", params=["tiny", "small"])
def golden(request):
    return dict(np.load(os.path.join(GOLDEN, f"bprmf_{request.param}.npz")))


@pytest.fixture(scope="session")
def golden_small():
    return dict(np.load(os.path.join(GOLDEN, "bprmf_small.npz")))


@pytest.fixture(scope="session")
def golden_tiny():
    return dict(np.load(os.path.join(GOLDEN, "bprmf_tiny.npz")))
