"""CPU: ResnetBlock recompute of the video autoencoder (tae.enable_training(..., recompute=True)) without a device: the
opt-in flags, the refusals that still fire with recompute on, and the C entry point vqb_gn_silu_apply (declaration,
export, argument validation, no device)."""
import ctypes
import os

import pytest
import torch

from oracle import tae_oracle as TO

EINVAL, ENODEVICE = -1, -2
SMALL = TO.TAEConfig(ch=32, ch_mult=(1, 8), num_res_blocks=1, z_channels=4, resolution=16)


def _blocks(m):
    import tae

    return [s for s in m.modules() if isinstance(s, tae.ResnetBlock)]


def test_recompute_flag_on_every_resnet_block_and_state_dict_unchanged():
    import tae

    torch.manual_seed(5)
    m = tae.TVAE(**SMALL.kwargs())
    torch.manual_seed(5)
    ref = tae.TVAE(**SMALL.kwargs())
    assert tae.enable_training(m, recompute=True) is m
    blocks = _blocks(m)
    levels, nrb = len(SMALL.ch_mult), SMALL.num_res_blocks
    assert len(blocks) == (levels * nrb + 2) + (2 + levels * (nrb + 1))  # encoder levels + mid, decoder mid + levels
    assert all(b._vqb_recompute for b in blocks)
    assert all(getattr(s, "_vqb_training", False) for s in m.modules())
    sd, sr = m.state_dict(), ref.state_dict()
    assert list(sd) == list(sr) and all(torch.equal(sd[k], sr[k]) for k in sd)
    tae.enable_training(m, False)
    assert not any(getattr(s, "_vqb_training", False) or getattr(s, "_vqb_recompute", False) for s in m.modules())


def test_default_opt_in_does_not_recompute_and_partial_opt_in_composes():
    import tae

    m = tae.enable_training(tae.TVAE(**SMALL.kwargs()), recompute=True)
    tae.enable_training(m)  # the default keeps today's path
    assert not any(b._vqb_recompute for b in _blocks(m))
    tae.enable_training(m.decoder, recompute=True)
    assert all(b._vqb_recompute for b in _blocks(m.decoder))
    assert not any(b._vqb_recompute for b in _blocks(m.encoder))
    assert all(s._vqb_training for s in m.modules())


def test_refusals_still_fire_with_recompute():
    import tae

    x = torch.zeros(1, 3, 4, 16, 24)
    m = tae.enable_training(tae.TVAE(**SMALL.kwargs()), enabled=False, recompute=True)
    with pytest.raises(RuntimeError, match="no_grad") as e:
        m(x)  # not opted in
    assert "enable_training" in str(e.value)
    blk = m.encoder.down[0].block[0]
    with pytest.raises(RuntimeError, match="no_grad"):
        blk(torch.zeros(1, 32, 2, 4, 4))
    tae.enable_training(m.bfloat16(), recompute=True)
    with pytest.raises(RuntimeError, match="bfloat16.*inference-only"):
        m(x.bfloat16())
    with pytest.raises(RuntimeError, match="bfloat16.*inference-only"):
        blk(torch.zeros(1, 32, 2, 4, 4, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="float16"):
        m.half()(x.half())


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    return native.load()


def test_gn_silu_apply_is_declared_and_exported(lib):
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vqb200.h")).read()
    assert "int vqb_gn_silu_apply(const void* x, void* y, const float* gamma, const float* beta, const float* mr, " \
           "int N, int HW,\n                      int C, int G, int silu, void* stream);" in hdr
    assert hasattr(lib, "vqb_gn_silu_apply")
    assert lib.vqb_version() >= 103


def test_gn_silu_apply_validates_and_fails_without_device(lib):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    f = lib.vqb_gn_silu_apply
    bads = [
        lambda: f(None, p, p, p, p, 1, 64, 64, 32, 1, None),   # null x
        lambda: f(p, None, p, p, p, 1, 64, 64, 32, 1, None),   # null y
        lambda: f(p, p, None, p, p, 1, 64, 64, 32, 1, None),   # null gamma
        lambda: f(p, p, p, p, None, 1, 64, 64, 32, 1, None),   # null mr
        lambda: f(p, p, p, p, p, 1, 64, 60, 30, 1, None),      # C % 8
        lambda: f(p, p, p, p, p, 1, 64, 64, 48, 1, None),      # C % G
        lambda: f(p, p, p, p, p, 1, 64, 4096, 32, 1, None),    # C above the limit
        lambda: f(p, p, p, p, p, 1, 64, 64, 0, 1, None),       # G = 0
        lambda: f(p, p, p, p, p, 1, 64, 64, 32, 2, None),      # silu not 0/1
        lambda: f(p, p, p, p, p, 0, 64, 64, 32, 1, None),      # N = 0
        lambda: f(p + 8, p, p, p, p, 1, 64, 64, 32, 1, None),  # x misaligned
        lambda: f(p, p + 2, p, p, p, 1, 64, 64, 32, 1, None),  # y misaligned
        lambda: f(p, p, p, p, p + 2, 1, 64, 64, 32, 1, None),  # mr misaligned
    ]
    for i, bad in enumerate(bads):
        assert bad() == EINVAL, i
        assert b"vqb_gn_silu_apply" in lib.vqb_last_error(), i
    for C in (64, 256, 1024, 2048):
        assert f(p, p, p, p, p, 2, 37, C, 32, 0, None) == ENODEVICE, C
        assert b"sm_90" in lib.vqb_last_error()
