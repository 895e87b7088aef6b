"""CPU: per-frame image losses on [B, 3, T, H, W] clips. The folded-frame oracle equals the per-image oracle frame by
frame; LPIPS / PatchDiscriminator refuse bad clip calls on the host before any launch; the clip boundary entry points of
include/vqb200.h validate their arguments (VQB_EINVAL) and, given valid ones, fail with VQB_ENODEVICE without an sm_90
device; VideoTrainer's frame draw follows torch's CPU generator."""
import ctypes
import os

import pytest
import torch

from helpers import seeded_sd
from oracle import clip_loss_oracle as CO
from oracle import lpips_oracle as LP
from oracle import seeded

EINVAL, ENODEVICE = -1, -2


@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    return native.load()


@pytest.mark.parametrize("frames", [None, [[2, 0], [1, 2]]])
def test_folded_oracle_equals_the_image_oracle_per_frame(frames):
    B, T = 2, 3
    x = seeded.tensor("clip_host/x", (B, 3, T, 32, 32), 1.0, "uniform")
    y = seeded.tensor("clip_host/y", (B, 3, T, 32, 32), 1.0, "uniform")
    sel = [list(range(T))] * B if frames is None else frames
    lsd = seeded_sd(LP.lpips_state_dict_shapes(), "lpips")
    psd = seeded_sd(LP.patchd_state_dict_shapes(), "patchd")
    with torch.no_grad():
        got_l = CO.lpips_clip(lsd, x, y, frames)
        got_p = CO.patchd_clip(psd, x, frames)
        want_l = torch.cat([LP.lpips_forward(lsd, x[b:b + 1, :, t], y[b:b + 1, :, t]) for b in range(B) for t in sel[b]])
        want_p = torch.cat([LP.patchd_forward(psd, x[b:b + 1, :, t]) for b in range(B) for t in sel[b]])
    assert got_l.shape == (B * len(sel[0]), 1, 1, 1) and got_p.shape == (B * len(sel[0]), 4)
    assert torch.equal(CO.fold_frames(x, frames)[1], x[0, :, sel[0][1]])
    torch.testing.assert_close(got_l, want_l, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(got_p, want_p, rtol=1e-5, atol=1e-6)


def _modules():
    import utils

    return utils.LPIPS().eval(), utils.PatchDiscriminator()


@pytest.mark.parametrize("case, match", [
    ("duplicate", "duplicate"),
    ("out_of_range", "outside"),
    ("negative", "outside"),
    ("rows", r"\[B, T'\]"),
    ("too_many", r"\[B, T'\]"),
    ("float", "integers"),
    ("channels", "channels"),
    ("target_shape", "differs"),
    ("target_4d", "differs"),
    ("frames_on_images", "clips"),
])
def test_bad_clip_calls_are_refused_before_any_launch(lib, case, match):
    import native

    lp, pd = _modules()
    x = torch.zeros(2, 3, 4, 32, 32)
    tgt, frames = x, None
    if case == "duplicate":
        frames = [[0, 1], [3, 3]]
    elif case == "out_of_range":
        frames = [[0, 4], [1, 2]]
    elif case == "negative":
        frames = torch.tensor([[0, -1], [1, 2]])
    elif case == "rows":
        frames = [[0, 1]]
    elif case == "too_many":
        frames = [[0, 1, 2, 3, 0], [0, 1, 2, 3, 1]]
    elif case == "float":
        frames = torch.tensor([[0.0, 1.0], [1.0, 2.0]])
    elif case == "channels":
        x = tgt = torch.zeros(2, 4, 4, 32, 32)
    elif case == "target_shape":
        tgt = torch.zeros(2, 3, 3, 32, 32)
    elif case == "target_4d":
        tgt = torch.zeros(2, 3, 32, 32)
    elif case == "frames_on_images":
        x = tgt = torch.zeros(2, 3, 32, 32)
        frames = [[0], [0]]
    n0 = native.launch_count()
    with pytest.raises(ValueError, match=match):
        lp(x, tgt, frames=frames)
    if case not in ("target_shape", "target_4d"):
        with pytest.raises(ValueError, match=match):
            pd(x, frames=frames)
    assert native.launch_count() == n0


def test_frame_selection_is_flattened_in_clip_order():
    import ops

    sel, k = ops.clip_frame_selection(torch.tensor([[3, 0], [1, 2]]), 2, 4)
    assert k == 2 and sel.dtype == torch.int32 and sel.tolist() == [3, 0, 1, 2]
    assert ops.clip_frame_selection(None, 2, 4) == (None, 4)


def clip_calls(p):
    """(name, call with valid arguments, [calls with invalid arguments]) for every clip boundary entry point."""
    s = p  # any non-null pointer stands for shift / inv_scale / the frame list
    return [
        ("vqb_ncthw_frames_to_nhwc_pad",
         lambda L: L.vqb_ncthw_frames_to_nhwc_pad(p, p, 2, 3, 4, 8, 8, 8, 1, p, 2, s, s, None),
         [lambda L: L.vqb_ncthw_frames_to_nhwc_pad(None, p, 2, 3, 4, 8, 8, 8, 1, p, 2, s, s, None),
          lambda L: L.vqb_ncthw_frames_to_nhwc_pad(p, p, 2, 3, 4, 8, 8, 8, 1, None, 2, s, s, None),  # Tsel != T
          lambda L: L.vqb_ncthw_frames_to_nhwc_pad(p, p, 2, 3, 4, 8, 8, 8, 1, p, 5, s, s, None),  # Tsel > T
          lambda L: L.vqb_ncthw_frames_to_nhwc_pad(p, p, 2, 3, 4, 8, 8, 8, -1, p, 2, s, s, None),
          lambda L: L.vqb_ncthw_frames_to_nhwc_pad(p, p, 2, 3, 4, 8, 8, 8, 1, p, 2, s, None, None)]),
        ("vqb_ncthw_frames_to_nhwc_pad_bf16",
         lambda L: L.vqb_ncthw_frames_to_nhwc_pad_bf16(p, p, 2, 3, 4, 8, 8, 8, 1, None, 4, s, s, None),
         [lambda L: L.vqb_ncthw_frames_to_nhwc_pad_bf16(p, None, 2, 3, 4, 8, 8, 8, 1, None, 4, s, s, None),
          lambda L: L.vqb_ncthw_frames_to_nhwc_pad_bf16(p, p, 2, 9, 4, 8, 8, 8, 1, None, 4, s, s, None)]),  # Cpad < C
        ("vqb_ncthw_frames_to_nhwc",
         lambda L: L.vqb_ncthw_frames_to_nhwc(p, p, 2, 3, 4, 8, 8, 8, p, 1, None, None, None),
         [lambda L: L.vqb_ncthw_frames_to_nhwc(p, p, 2, 3, 0, 8, 8, 8, p, 1, None, None, None),
          lambda L: L.vqb_ncthw_frames_to_nhwc(p, p, 40000, 3, 4, 8, 8, 8, None, 4, None, None, None)]),  # grid
        ("vqb_ncthw_frames_to_nhwc_bf16",
         lambda L: L.vqb_ncthw_frames_to_nhwc_bf16(p, p, 1, 3, 4, 8, 8, 16, p, 3, s, s, None),
         [lambda L: L.vqb_ncthw_frames_to_nhwc_bf16(p, p, 1, 3, 4, 8, 8, 12, p, 3, s, s, None)]),  # Cpad % 8
        ("vqb_nhwc_pad_frames_to_ncthw",
         lambda L: L.vqb_nhwc_pad_frames_to_ncthw(p, p, 2, 3, 4, 8, 8, 8, 1, p, 2, s, None),
         [lambda L: L.vqb_nhwc_pad_frames_to_ncthw(p, None, 2, 3, 4, 8, 8, 8, 1, p, 2, s, None),
          lambda L: L.vqb_nhwc_pad_frames_to_ncthw(p, p, 2, 3, 4, 8, 8, 8, 1, p, 0, s, None)]),
        ("vqb_nhwc_frames_to_ncthw",
         lambda L: L.vqb_nhwc_frames_to_ncthw(p, p, 2, 3, 4, 8, 8, 8, None, 4, None, None),
         [lambda L: L.vqb_nhwc_frames_to_ncthw(p, p, 2, 3, 4, 8, -8, 8, None, 4, None, None)]),
    ]


def test_clip_entry_points_are_declared_and_exported(lib):
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vqb200.h")).read()
    for name, _, _ in clip_calls(0):
        assert f"int {name}(" in hdr, name
        assert hasattr(lib, name), name


def test_clip_entry_points_validate_then_need_a_device(lib):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.addressof(buf)
    for name, good, bads in clip_calls(p):
        for i, bad in enumerate(bads):
            assert bad(lib) == EINVAL, (name, i)
            assert name.encode() in lib.vqb_last_error(), (name, i)
        assert good(lib) == ENODEVICE, name
        assert b"sm_90" in lib.vqb_last_error(), name


def test_null_pointer_messages_name_the_argument(lib):
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 64)()
    p = ctypes.addressof(buf)
    assert lib.vqb_ncthw_frames_to_nhwc(None, p, 1, 3, 1, 8, 8, 8, None, 1, None, None, None) == EINVAL
    assert b"input" in lib.vqb_last_error()
    assert lib.vqb_nhwc_frames_to_ncthw(p, None, 1, 3, 1, 8, 8, 8, None, 1, None, None) == EINVAL
    assert b"output" in lib.vqb_last_error()


def test_video_trainer_draws_distinct_frames_from_the_cpu_generator():
    import tae_trainer

    tr = tae_trainer.VideoTrainer.__new__(tae_trainer.VideoTrainer)
    tr.perceptual_frames = 3
    torch.manual_seed(5)
    a = tr.draw_frames(4, 8)
    torch.manual_seed(5)
    b = tr.draw_frames(4, 8)
    assert torch.equal(a, b) and a.shape == (4, 3)
    assert all(len(set(r)) == 3 and all(0 <= v < 8 for v in r) for r in a.tolist())
    tr.perceptual_frames = None
    assert tr.draw_frames(4, 8) is None
    tr.perceptual_frames = 9
    with pytest.raises(ValueError, match="exceeds"):
        tr.draw_frames(4, 8)


def test_video_trainer_fold_matches_the_oracle_fold():
    import tae_trainer

    x = seeded.tensor("clip_host/fold", (2, 3, 5, 4, 6))
    f = torch.tensor([[4, 1], [0, 3]])
    assert torch.equal(tae_trainer.fold_frames(x, f), CO.fold_frames(x, f))
    assert torch.equal(tae_trainer.fold_frames(x), CO.fold_frames(x))
