import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "deep-image-prior_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    try:
        import torch
        # the GPU box exposes 100+ logical cores; torch-CPU (the oracle) is fastest with a handful of threads
        torch.set_num_threads(min(8, os.cpu_count() or 1))
    except Exception:
        pass
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
