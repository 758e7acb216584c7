import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is visible, so a bare
    `pytest tests/` works on a machine without a GPU.  `-m gpu` on a GPU box runs them."""
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
