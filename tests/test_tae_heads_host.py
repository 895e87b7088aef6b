"""CPU: which attention head sizes the video autoencoder accepts. Heads of 8 to 112 channels in steps of 8 (tae.AttnBlock
in_channels a multiple of 64 up to 896) pass the host checks of tae.AttnBlock and ops; every other size is refused with
NotImplementedError naming it, before anything is launched. The C ABI refuses the same sizes with EINVAL and a message
naming the head_dim, and returns ENODEVICE for every accepted size when no sm_90 device is present."""
import ctypes

import pytest
import torch

from test_tae_host import EINVAL, ENODEVICE, lib  # noqa: F401  (module fixture)

ACCEPTED = list(range(8, 113, 8))
REFUSED = [4, 12, 20, 60, 120, 128, 136, 256]


def test_ops_head_dims_are_the_multiples_of_8_up_to_112():
    import ops

    assert ops.ATTN_HEAD_DIMS == tuple(ACCEPTED)


@pytest.mark.parametrize("C", [8 * hd for hd in ACCEPTED])
def test_attn_block_accepts(C):
    import tae

    blk = tae.AttnBlock(C)
    assert blk.head_dim == C // 8
    blk._check_heads()


@pytest.mark.parametrize("C", [8 * hd for hd in REFUSED])
def test_attn_block_refuses_naming_the_head_size(C):
    import tae

    blk = tae.AttnBlock(C)
    with pytest.raises(NotImplementedError, match=f"heads of {C / 8:g} channels"):
        blk._check_heads()


@pytest.mark.parametrize("hd", REFUSED)
def test_ops_refuses_before_any_launch(hd, lib):  # noqa: F811
    """A CPU tensor: an accepted size would fail later, at the device; a refused one never gets there."""
    import native
    import ops

    n0 = native.launch_count()
    qkv = torch.zeros(1, 1, 2, 2, 3 * 8 * hd, dtype=torch.bfloat16)
    for fn in (ops.attention_hd, ops.attention_hd_train):
        with pytest.raises(NotImplementedError, match=f"heads of {hd} channels"):
            fn(qkv, 8, hd)
    assert native.launch_count() == n0


@pytest.mark.parametrize("ch,ch_mult,head_dim", [(32, (1, 2, 4, 4), 16), (96, (1, 2, 4, 4), 48),
                                                 (224, (1, 4), 112), (32, (1, 2), 8), (160, (1, 2), 40)])
def test_tvae_widths_pass_the_head_check(ch, ch_mult, head_dim):
    import tae

    m = tae.TVAE(resolution=64, in_channels=3, ch=ch, out_ch=3, ch_mult=list(ch_mult), num_res_blocks=1, z_channels=4)
    for blk in (m.encoder.mid.attn_1, m.decoder.mid.attn_1):
        assert blk.head_dim == head_dim
        blk._check_heads()


def test_abi_validates_head_dim_without_device(lib):  # noqa: F811
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    for hd in REFUSED:
        C = 8 * hd
        assert lib.vqb_attn_fwd_hd(p, p, p, 1, 64, C, hd, None) == EINVAL, hd
        assert f"head_dim={hd}".encode() in lib.vqb_last_error(), hd
        assert lib.vqb_attn_bwd_hd(p, p, p, p, p, p, 1, 64, C, hd, None) == EINVAL, hd
        assert f"head_dim={hd}".encode() in lib.vqb_last_error(), hd
    for hd in ACCEPTED:
        C = 8 * hd
        assert lib.vqb_attn_fwd_hd(p, p, p, 1, 64, C, hd, None) == ENODEVICE, hd
        assert b"sm_90" in lib.vqb_last_error(), hd
        assert lib.vqb_attn_bwd_hd(p, p, p, p, p, p, 1, 64, C, hd, None) == ENODEVICE, hd
        assert b"sm_90" in lib.vqb_last_error(), hd
        # C not a multiple of the head size: refused before the device check
        assert lib.vqb_attn_fwd_hd(p, p, p, 1, 64, C + 4, hd, None) == EINVAL, hd
        assert lib.vqb_attn_bwd_hd(p, p, p, p, p, p, 1, 64, C + 4, hd, None) == EINVAL, hd
