import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on a GPU host)")
    config.addinivalue_line("markers", "slow: takes more than a few seconds on CPU")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a host without a CUDA device skips the `gpu` tests instead of failing at the first of them."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (run on a GPU host: pytest -m gpu)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
