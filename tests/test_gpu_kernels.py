"""GPU (-m gpu): kernel-level parity of the C ABI entry points against plain PyTorch fp32 references
(tools/gpu_probe.py holds the cases: wgmma conv fwd/dgrad/stride-2 with every epilogue operand, wgrad,
GroupNorm/SiLU, layout, pooling)."""
import importlib
import os
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def probe():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    return importlib.import_module("gpu_probe")


@pytest.mark.parametrize("group", ["gemm", "conv", "conv2", "wgrad", "elem", "lpips", "up", "stats", "fat"])
def test_kernel_group(probe, group):
    assert getattr(probe, "group_" + group)(), f"kernel parity group {group} has failures (see stdout)"

