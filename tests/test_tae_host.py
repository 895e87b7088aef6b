"""CPU: the video autoencoder (tae.py) path without a device. The 3-D conv plans emulated with the documented kernel
semantics of vqb_conv3d_gemm against F.conv3d, the oracle against the reference fixture, the seeded initialisation
against the reference's digests, the new C ABI, and the host-side refusals."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import plans
from helpers import golden, rel_l2, t
from oracle import seeded
from oracle import tae_oracle as TO

EINVAL, ENODEVICE = -1, -2


def emulate_conv3d(g: plans.ConvGeom3d, a: torch.Tensor, wp: torch.Tensor, Cout: int):
    """include/vqb200.h semantics of vqb_conv3d_gemm: out[n,t,h,w,co] = sum_tap sum_c
    view_tap[n, t+dt, h+dh, w+dw, c] * wp[co][tap][c]; reads outside a view are zero. a: flat fp32 buffer of the A
    tensor; wp [Cout][taps][C]."""
    flat = torch.cat([a.reshape(-1), torch.zeros(g.C)])  # one zero row past the end stands for masked reads
    zero = flat.numel() - g.C
    n, tt, hh, ww = torch.meshgrid(torch.arange(g.N), torch.arange(g.To), torch.arange(g.Ho), torch.arange(g.Wo),
                                   indexing="ij")
    out = torch.zeros(g.N, g.To, g.Ho, g.Wo, Cout)
    for i, (v, dw, dh, dt) in enumerate(g.taps):
        vw = g.views[v]
        ts, hs, ws = tt + dt, hh + dh, ww + dw
        ok = (ts >= 0) & (ts < vw.Tv) & (hs >= 0) & (hs < vw.Hv) & (ws >= 0) & (ws < vw.Wv) & (n < vw.Nv)
        off = vw.offset + n * vw.sn + ts * vw.st + hs * vw.sh + ws * vw.sw
        off = torch.where(ok, off, torch.full_like(off, zero))
        rows = flat[off.reshape(-1, 1) + torch.arange(g.C)]  # [voxels, C]
        out += (rows @ wp[:, i, :].T).reshape(out.shape)
    return out


def pack3(w, tapmap):
    Cout, Cin = w.shape[:2]
    return w.reshape(Cout, Cin, -1)[:, :, tapmap].permute(0, 2, 1).contiguous()


def pack3_fold(w, masks):
    Cout, Cin = w.shape[:2]
    wf = w.reshape(Cout, Cin, 27)
    cols = [sum(wf[:, :, b] for b in range(27) if (m >> b) & 1) for m in masks]
    return torch.stack(cols, 1)  # [Cout][slots][Cin]


def test_geom3_s1_matches_conv3d():
    torch.manual_seed(0)
    N, T, H, W, C, Co = 2, 3, 5, 7, 8, 4
    x, w = torch.randn(N, T, H, W, C), torch.randn(Co, C, 3, 3, 3)
    g = plans.geom3_s1(N, T, H, W, C)
    assert len(g.taps) == 27 and sorted(g.tapmap) == list(range(27))
    out = emulate_conv3d(g, x, pack3(w, g.tapmap), Co)
    ref = F.conv3d(x.permute(0, 4, 1, 2, 3), w, padding=1).permute(0, 2, 3, 4, 1)
    assert torch.allclose(out, ref, atol=1e-4)


def test_geom3_s2_matches_padded_stride2_conv():
    """Downsample (tae.py:100-104): F.pad(x, (0,1,0,1,0,1)) then 3x3x3 stride 2; the pad planes are the zero fill."""
    torch.manual_seed(1)
    N, T, H, W, C, Co = 2, 4, 6, 10, 8, 5
    x, w = torch.randn(N, T, H, W, C), torch.randn(Co, C, 3, 3, 3)
    g = plans.geom3_s2(N, T, H, W, C)
    assert len(g.views) == 8 and len(g.taps) == 27
    out = emulate_conv3d(g, x, pack3(w, g.tapmap), Co)
    ref = F.conv3d(F.pad(x.permute(0, 4, 1, 2, 3), (0, 1, 0, 1, 0, 1)), w, stride=2).permute(0, 2, 3, 4, 1)
    assert out.shape == ref.shape and torch.allclose(out, ref, atol=1e-4)


def test_geom3_up_phases_match_interpolate_then_conv():
    """Upsample (tae.py:114-116): the 8 folded 2x2x2-tap phases equal conv3d(interpolate(x, 2, nearest), padding 1)."""
    torch.manual_seed(2)
    N, t_, h, w_, C, Co = 1, 3, 5, 7, 8, 6
    x, w = torch.randn(N, t_, h, w_, C), torch.randn(Co, C, 3, 3, 3)
    out = torch.zeros(N, 2 * t_, 2 * h, 2 * w_, Co)
    macs = 0
    for pt in range(2):
        for ph in range(2):
            for pw in range(2):
                g = plans.geom3_up_fwd(N, t_, h, w_, C, pt, ph, pw)
                assert len(g.taps) == 8 and all(0 < m < (1 << 27) for m in g.tapmask)
                out[:, pt::2, ph::2, pw::2] = emulate_conv3d(g, x, pack3_fold(w, g.tapmask), Co)
                macs += len(g.taps)
    up = F.interpolate(x.permute(0, 4, 1, 2, 3), scale_factor=2.0, mode="nearest")
    ref = F.conv3d(up, w, padding=1).permute(0, 2, 3, 4, 1)
    assert torch.allclose(out, ref, atol=1e-3)
    assert macs == 64  # per low-res voxel: 64 folded taps instead of 8 x 27 = 216 (8/27 of the MACs)


def test_phase_output_strides_address_the_subgrid():
    t_, h, w_, Cop = 2, 3, 5, 16
    on, ot, oh, ow, oc = plans.up3_out_strides(t_, h, w_, Cop)
    full = torch.arange(2 * t_ * 2 * h * 2 * w_ * Cop).view(2 * t_, 2 * h, 2 * w_, Cop)
    for pt, ph, pw in [(0, 0, 0), (1, 0, 1), (1, 1, 1)]:
        base = ((pt * 2 * h + ph) * 2 * w_ + pw) * Cop
        a, b, c = 1, 2, 3
        assert full[pt::2, ph::2, pw::2][a, b, c, 5] == base + a * ot + b * oh + c * ow + 5 * oc
    assert on == full.numel()


def _small_sd():
    import tae

    m = tae.TVAE(**TO.TAEConfig(ch=32, ch_mult=(1, 8), num_res_blocks=1, z_channels=4, resolution=16).kwargs())
    return seeded.fill_state_dict(m.state_dict(), "tae_small")


def test_oracle_reproduces_reference_fixture():
    gd = golden("tae_small")
    cfg = TO.TAEConfig(ch=32, ch_mult=(1, 8), num_res_blocks=1, z_channels=4, resolution=16)
    with torch.no_grad():
        decz, z = TO.forward(_small_sd(), t(gd["x"]), t(gd["eps"]), cfg)
    assert rel_l2(z, gd["z"]) < 1e-4
    assert rel_l2(decz, gd["decz"]) < 1e-4


def test_seeded_init_matches_reference_bit_for_bit():
    import tae

    gd = golden("tae_init_seed123")
    torch.manual_seed(123)
    sd = tae.TVAE(resolution=32, in_channels=3, ch=32, out_ch=3, ch_mult=[1, 2], num_res_blocks=2,
                  z_channels=4).state_dict()
    keys = sorted(sd)
    assert keys == [str(k) for k in gd["keys"]]
    for i, k in enumerate(keys):
        shp = [s for s in gd["shapes"][i] if s >= 0]
        assert list(sd[k].shape) == shp, k
        assert hashlib.sha256(sd[k].detach().contiguous().numpy().tobytes()).hexdigest() == str(gd["sha256"][i]), k


def test_module_surface_matches_reference_names():
    import inspect

    import tae

    for name in ("swish", "AttnBlock", "ResnetBlock", "Downsample", "Upsample", "Encoder", "Decoder",
                 "DiagonalGaussian", "TVAE"):
        assert hasattr(tae, name), name
    assert list(inspect.signature(tae.TVAE.__init__).parameters) == [
        "self", "resolution", "in_channels", "ch", "out_ch", "ch_mult", "num_res_blocks", "z_channels"]


def test_refusals_before_any_launch_on_the_host():
    import tae

    m = tae.TVAE(**TO.TAEConfig(ch=32, ch_mult=(1, 8), num_res_blocks=1, z_channels=4, resolution=16).kwargs())
    x = torch.zeros(1, 3, 4, 16, 24)
    with pytest.raises(RuntimeError, match="no_grad"):
        m(x)  # grad enabled, parameters require grad
    with torch.no_grad(), pytest.raises(ValueError, match=r"\(1, 3, 5, 16, 24\)"):
        m(torch.zeros(1, 3, 5, 16, 24))
    with torch.no_grad(), pytest.raises(RuntimeError, match="float16"):
        m.half()(x.half())
    big = tae.AttnBlock(1024)  # heads of 128
    with torch.no_grad(), pytest.raises(NotImplementedError, match="128"):
        big(torch.zeros(1, 1024, 1, 2, 2))


# ---------------------------------------------------------------------------------------------------- C ABI
@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    return native.load()


def _desc(bad=None):
    g = plans.geom3_s1(1, 2, 4, 4, 8)
    d = plans.conv3d_desc(g, 16, plans.nthwc_strides(2, 4, 4, 16))
    if bad == "flags":
        d.flags = 4  # VQB_EPI_RELU: not on the rank-5 epilogue
    elif bad == "taps":
        d.ntaps = 28
    elif bad == "view":
        d.taps[3].view = 1
    return d


def calls(p):
    return [
        ("vqb_conv3d_gemm",
         lambda L: L.vqb_conv3d_gemm(_desc(), p, p, None, None, p, None),
         [lambda L: L.vqb_conv3d_gemm(_desc("flags"), p, p, None, None, p, None),
          lambda L: L.vqb_conv3d_gemm(_desc("taps"), p, p, None, None, p, None),
          lambda L: L.vqb_conv3d_gemm(_desc("view"), p, p, None, None, p, None),
          lambda L: L.vqb_conv3d_gemm(_desc(), p, None, None, None, p, None)]),
        ("vqb_attn_fwd_hd",
         lambda L: L.vqb_attn_fwd_hd(p, p, p, 1, 64, 256, 32, None),
         [lambda L: L.vqb_attn_fwd_hd(p, p, p, 1, 64, 1024, 128, None),
          lambda L: L.vqb_attn_fwd_hd(p, p, p, 1, 64, 200, 32, None)]),
        ("vqb_gauss_reparam",
         lambda L: L.vqb_gauss_reparam(p, p, p, 1, 4, 64, 1, None),
         [lambda L: L.vqb_gauss_reparam(p, p, p, 1, 0, 64, 1, None),
          lambda L: L.vqb_gauss_reparam(p, None, p, 1, 4, 64, 0, None)]),
    ]


def test_video_entry_points_are_declared_and_exported(lib):
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vqb200.h")).read()
    for name, _, _ in calls(0):
        assert f"int {name}(" in hdr, name
        assert hasattr(lib, name), name


def test_video_entry_points_validate_and_fail_without_device(lib):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    for name, good, bads in calls(p):
        for bad in bads:
            assert bad(lib) == EINVAL, name
        assert good(lib) == ENODEVICE, name
        assert b"sm_90" in lib.vqb_last_error(), name
    assert lib.vqb_attn_fwd_hd(p, p, p, 1, 64, 1024, 128, None) == EINVAL
    assert b"head_dim=128" in lib.vqb_last_error()


def test_struct_sizes_match_the_header():
    import native

    assert ctypes.sizeof(native.VqbView3d) == 8 + 4 * 4 + 4 * 8
    assert ctypes.sizeof(native.VqbTap3d) == 16
    assert ctypes.sizeof(native.VqbConv3dDesc) == 10 * 4 + 5 * 8 + 8 * 56 + 27 * 16
    assert ctypes.sizeof(native.VqbConvDesc) == 10 * 4 + 4 * 8 + 16 * 48 + 16 * 16  # unchanged
    assert ctypes.sizeof(native.VqbView) == 48 and ctypes.sizeof(native.VqbTap) == 16
    assert [f for f, _ in native.VqbConv3dDesc._fields_][:10] == ["C", "Cout", "N", "T", "H", "W", "nviews", "ntaps",
                                                                 "flags", "out_f32"]


def test_flop_count_of_the_reference_main_config():
    """Algorithmic FLOPs of the folded plan for tae.py's __main__ config: 18.0 TFLOP as written, minus about 3 for the
    folded up-sampling."""
    f = TO.flops(TO.TAEConfig(), 1, 48, 256, 256)
    assert 14.0e12 < f < 15.5e12, f
