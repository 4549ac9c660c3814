import asyncio
import functools
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")
    config.addinivalue_line("markers", "slow: multi-process / long-running")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        have_gpu = torch.cuda.is_available()
        n_gpu = torch.cuda.device_count() if have_gpu else 0
    except Exception:
        have_gpu, n_gpu = False, 0
    skip_gpu = pytest.mark.skip(reason="no CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
    for item in items:
        if "gpu" in item.keywords and not have_gpu:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and n_gpu < 2:
            item.add_marker(skip_multi)


def run_async(fn):
    """Run an ``async def`` test on a fresh event loop (no pytest-asyncio here)."""
    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        return asyncio.run(asyncio.wait_for(fn(*args, **kwargs), timeout=60))
    return wrapper
