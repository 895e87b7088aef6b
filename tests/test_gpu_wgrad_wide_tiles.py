"""The 256-column tile of the weight-gradient GEMM (csrc/wgrad_gemm.cu): the element-wise fp64 bound, the guard bands
and the run-twice bit equality of test_gpu_kernel_bounds.py at shapes whose (tap, channel) columns divide by 256,
including tiles that hold two taps and splits that get no pixel box."""
import pytest

import test_gpu_kernel_bounds as KB
from test_gpu_kernel_bounds import lib  # noqa: F401  (module fixture: loads the library, skips without an sm_90 device)

pytestmark = pytest.mark.gpu


WGRAD_CASES = [
    # kind, (N, H, W) of x, C, Cout, ksplit, Cin, accumulate  (columns = taps * C64, all multiples of 256)
    ("s1", (2, 12, 10), 256, 136, 3, 256, 0),
    ("s1", (1, 9, 9), 512, 72, 2, 512, 1),
    ("p1", (3, 8, 8), 512, 256, 5, 512, 0),  # 3 pixel boxes, 5 splits: two splits contribute zeros
    ("up", (2, 6, 6), 128, 136, 3, 128, 0),  # 4 taps x 128 channels: every 256-column tile holds two taps
    ("s2", (2, 16, 12), 256, 72, 1, 250, 0),
    ("s1", (5, 8, 8), 256, 8, 5, 256, 0),  # one box per split
]


@pytest.mark.parametrize("kind,shp,C,Cout,ksplit,Cin,acc", WGRAD_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_wgrad_256_column_tiles_bounds(kind, shp, C, Cout, ksplit, Cin, acc):
    import ops

    ntaps = {"s1": 9, "s2": 9, "p1": 1, "up": 4}[kind]
    assert ops._wgrad_block_n(ntaps * C) * ops._wgrad_tile_blocks(ntaps * C) == 256
    KB.test_wgrad_bounds(kind, shp, C, Cout, ksplit, Cin, acc)
