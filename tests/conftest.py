import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
# Several logical ranks share ONE GPU in the gpu tests, each with its own sync stream whose device-side barrier kernel
# waits for the other ranks' kernels: give every stream its own hardware queue (default 8 connections would let one
# rank's kernels queue up behind another rank's waiting barrier). Must be set before CUDA initialises.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")
    config.addinivalue_line("markers", "slow: long-running stress variant")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_cuda = torch.cuda.is_available()
    except Exception:
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
