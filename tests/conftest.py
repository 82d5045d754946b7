import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture
def rpm_window():
    """Tests that run a router on the wall clock count admissions against per-minute rpm / tpm buckets; started in
    the last seconds of a minute they would straddle a window refill.  Wait the boundary out instead."""
    import time
    left = 60.0 - time.time() % 60.0
    if left < 8.0:
        time.sleep(left + 0.05)
    yield
