import os
import sys

# Virtual-rank tests launch one kernel per rank on separate streams of ONE device and those
# kernels wait for each other: give every stream its own hardware queue.  Must be set before
# CUDA initialises.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
# Lazy module loading loads a kernel on its first launch and may synchronise the context to do so: a first launch
# behind a virtual rank's kernel that spins on its peer would then wait for that peer forever.
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box)")


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
