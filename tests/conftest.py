import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "vqgan-training_b200")
for p in (PKG, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)
os.environ.setdefault("WANDB_MODE", "disabled")
os.environ.setdefault("VQB_OFFLINE", "1")  # do not try to download torchvision / LPIPS weights in tests


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90, H100) device; select with -m gpu")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
