"""The staged epilogue of the wgmma conv kernel (csrc/conv_gemm.cu). NHWC bf16 outputs with Cout % 64 == 0 take their
residual or ReLU mask from a shared-memory tile that TMA filled during the tile's MMAs, and leave through TMA tensor
stores of that tile. The stored bf16 must equal, bit for bit, the fragment-store path's fp32 NCHW output of the same
conv rounded to bf16 (the same fp32 value, rounded once). Every element outside the addressed output stays poisoned,
and the residual / mask buffer is read, never written. Cases cover every epilogue at BLOCK_N 64 and 128, ragged tiles,
column tiles with one 64-channel slab, strided outputs (stride-2 data-gradient classes, up-sampling phases), 1x1 and
2-tap launches, and CTAs that reuse each warpgroup's tile buffer at least three times."""
import inspect

import pytest
import torch

import test_gpu_kernel_bounds as KB
from test_gpu_kernel_bounds import check_stores
from test_gpu_kernel_bounds import lib  # noqa: F401  (module fixture: loads the library, skips without an sm_90 device)

pytestmark = pytest.mark.gpu


def staged_matches_fp32(kind, shp, C, Cout, epi):
    s = KB.build_conv2d(kind, shp, C, Cout, epi, "nhwc")
    f = KB.build_conv2d(kind, shp, C, Cout, epi.replace("+stats", ""), "nchw32")  # same seed: same operands
    name = f"conv {kind} {shp} C={C} Cout={Cout} {epi or 'plain'}"
    operands = inspect.getclosurevars(s.launch).nonlocals
    reads = [operands[k] for k in ("res", "mask") if operands[k] is not None]
    before = [g.bits() for g in reads]
    out, _ = s.launch()
    ref, _ = f.launch()
    check_stores(out, s.idx, name + " staged stores")
    for g, b in zip(reads, before):
        assert torch.equal(g.bits(), b), f"{name}: the residual / mask buffer was written"
    got = out.body[s.idx].view(torch.int16)
    want = ref.body[f.idx].to(torch.bfloat16).view(torch.int16)
    diff = (got != want).nonzero()
    assert diff.numel() == 0, f"{name}: {diff.shape[0]} stored values differ from the rounded fp32 output " \
                              f"(first at {diff[0].tolist()})"


EPIS = ("", "bias", "bias+res", "bias+res+stats", "relu", "mask")


@pytest.mark.parametrize("epi", EPIS, ids=lambda v: v or "plain")
@pytest.mark.parametrize("Cout", (64, 128))  # BLOCK_N 64 and 128
def test_staged_epilogues(Cout, epi):
    staged_matches_fp32("s1", (4, 16, 16), 64, Cout, epi)


@pytest.mark.parametrize("kind,shp,C,Cout,epi", [
    ("s1", (3, 5, 130), 72, 128, "bias+res"),          # ragged rows and columns of the pixel box
    ("s1", (2, 5, 3), 24, 64, "mask"),                 # boxes across images, ragged in both directions
    ("s1", (11, 4, 4), 136, 320, "bias+res+relu"),     # last column tile holds one 64-channel slab
    ("p1", (8, 64, 64), 64, 128, "bias"),              # 1x1, one K-chunk
    ("p1", (3, 1, 130), 136, 192, "res"),              # 1x1, one-row images, one-slab column tile
    ("dg200", (11, 8, 8), 64, 128, ""),                # stride-2 data-gradient classes: 1, 2 and 4 taps over
    ("dg201", (2, 64, 64), 128, 128, "mask"),          # a strided output
    ("dg210", (3, 2, 260), 72, 64, ""),
    ("dg211", (2, 6, 6), 136, 128, "mask"),
    ("up01", (11, 4, 4), 136, 128, "bias"),            # up-sampling phases: strided output, offset base
    ("up10", (2, 5, 3), 72, 64, "bias+res"),
], ids=lambda v: str(v).replace(" ", "") if not isinstance(v, str) else (v or "plain"))
def test_staged_shapes(kind, shp, C, Cout, epi):
    staged_matches_fp32(kind, shp, C, Cout, epi)


@pytest.mark.parametrize("Cout,epi", [(128, "bias+res+stats"), (64, "mask"), (128, "")])
def test_staged_buffer_reuse(Cout, epi):
    """8-9 tiles per CTA: each warpgroup refills and re-stores its tile buffer at least three times."""
    S = torch.cuda.get_device_properties(0).multi_processor_count
    staged_matches_fp32("s1", (8 * S + S // 2, 8, 16), 64, Cout, epi)  # one 128-pixel tile per image
