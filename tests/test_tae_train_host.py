"""CPU: the training path of the video autoencoder (tae.enable_training) without a device. The 3-D data- and
weight-gradient plans emulated with the documented kernel semantics (include/vqb200.h) against torch.autograd.grad of
F.conv3d in float64, the new C ABI (struct sizes, argument validation, no device), and the host-side refusals."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

import plans
from oracle import tae_oracle as TO
from test_tae_host import emulate_conv3d, pack3_fold

EINVAL, ENODEVICE = -1, -2
SMALL = TO.TAEConfig(ch=32, ch_mult=(1, 8), num_res_blocks=1, z_channels=4, resolution=16)


def _grads(fn, x, w, dy):
    x, w = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    return torch.autograd.grad(fn(x, w), (x, w), dy)


def _to_cl(x):  # NCTHW -> NTHWC
    return x.permute(0, 2, 3, 4, 1).contiguous()


def _gather(view, off_t, off_h, off_w, flat, C, N, To, Ho, Wo):
    """Rows [voxels, C] of `view` at (t + off_t, h + off_h, w + off_w) of the (N, To, Ho, Wo) grid; zero outside."""
    zero = flat.numel() - C
    n, tt, hh, ww = torch.meshgrid(torch.arange(N), torch.arange(To), torch.arange(Ho), torch.arange(Wo), indexing="ij")
    ts, hs, ws = tt + off_t, hh + off_h, ww + off_w
    ok = (ts >= 0) & (ts < view.Tv) & (hs >= 0) & (hs < view.Hv) & (ws >= 0) & (ws < view.Wv) & (n < view.Nv)
    off = view.offset + n * view.sn + ts * view.st + hs * view.sh + ws * view.sw
    off = torch.where(ok, off, torch.full_like(off, zero))
    return flat[off.reshape(-1, 1) + torch.arange(C)]


def emulate_wgrad3d(g: plans.ConvGeom3d, x: torch.Tensor, dy: torch.Tensor, Cout: int, dy_view=None):
    """include/vqb200.h semantics of vqb_wgrad3d_gemm: partial[co][tap][c] = sum over the dy voxel grid of
    dy_view[n, t, h, w, co] * X_view(tap)[n, t+dt, h+dh, w+dw, c]."""
    fx = torch.cat([x.reshape(-1), torch.zeros(g.C, dtype=x.dtype)])
    fy = torch.cat([dy.reshape(-1), torch.zeros(Cout, dtype=dy.dtype)])
    yv = dy_view if dy_view is not None else plans.dense_view3d(g.N, g.To, g.Ho, g.Wo, Cout)
    rows_y = _gather(yv, 0, 0, 0, fy, Cout, g.N, g.To, g.Ho, g.Wo)
    out = torch.zeros(Cout, len(g.taps), g.C, dtype=x.dtype)
    for i, (v, dw, dh, dt) in enumerate(g.taps):
        out[:, i, :] = rows_y.T @ _gather(g.views[v], dt, dh, dw, fx, g.C, g.N, g.To, g.Ho, g.Wo)
    return out


def reduce_tapmap(partial, tapmap, shape):
    """vqb_wgrad_reduce: slot -> tap of the OIDHW gradient."""
    Cout, Cin = shape[:2]
    gw = torch.zeros(Cout, Cin, 27, dtype=partial.dtype)
    for s, tap in enumerate(tapmap):
        gw[:, :, tap] += partial[:Cout, s, :Cin]
    return gw.reshape(shape)


def reduce_fold(partial, masks, shape):
    """vqb_wgrad_reduce_fold: slot s contributes to every tap in masks[s]."""
    Cout, Cin = shape[:2]
    gw = torch.zeros(Cout, Cin, 27, dtype=partial.dtype)
    for s, m in enumerate(masks):
        for tap in range(27):
            if (m >> tap) & 1:
                gw[:, :, tap] += partial[:Cout, s, :Cin]
    return gw.reshape(shape)


def pack3_t(w, tapmap):
    """Transposed (dgrad) packing: [Cin][taps][Cout]."""
    Cout, Cin = w.shape[:2]
    return w.reshape(Cout, Cin, -1)[:, :, tapmap].permute(1, 2, 0).contiguous()


def pack3_fold_t(w, masks):
    return pack3_fold(w.transpose(0, 1), masks)  # [Cin][slots][Cout]


# ------------------------------------------------------------------------------------------------ plans
@pytest.fixture
def f64():
    """emulate_conv3d accumulates in the default dtype: float64 for these comparisons."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


def test_s1_dgrad_and_wgrad_match_autograd(f64):
    torch.manual_seed(0)
    N, T, H, W, C, Co = 2, 3, 5, 7, 8, 16
    x, w = torch.randn(N, C, T, H, W, dtype=torch.float64), torch.randn(Co, C, 3, 3, 3, dtype=torch.float64)
    dy = torch.randn(N, Co, T, H, W, dtype=torch.float64)
    gx, gw = _grads(lambda x_, w_: F.conv3d(x_, w_, padding=1), x, w, dy)
    gd = plans.geom3_s1_dgrad(N, T, H, W, Co)
    assert len(gd.taps) == 27 and sorted(gd.tapmap) == list(range(27))
    ours = emulate_conv3d(gd, _to_cl(dy), pack3_t(w, gd.tapmap), C)
    assert torch.allclose(ours, _to_cl(gx), atol=1e-9)
    g = plans.geom3_s1(N, T, H, W, C)
    part = emulate_wgrad3d(g, _to_cl(x), _to_cl(dy), Co)
    assert torch.allclose(reduce_tapmap(part, g.tapmap, w.shape), gw, atol=1e-9)


def test_s2_dgrad_classes_and_wgrad_match_autograd(f64):
    """Downsample: F.pad(x, (0,1,0,1,0,1)) + stride-2 conv; the pad plane's gradient is dropped."""
    torch.manual_seed(1)
    N, T, H, W, C, Co = 2, 4, 6, 10, 8, 8
    x, w = torch.randn(N, C, T, H, W, dtype=torch.float64), torch.randn(Co, C, 3, 3, 3, dtype=torch.float64)
    dy = torch.randn(N, Co, T // 2, H // 2, W // 2, dtype=torch.float64)
    gx, gw = _grads(lambda x_, w_: F.conv3d(F.pad(x_, (0, 1, 0, 1, 0, 1)), w_, stride=2), x, w, dy)
    ours = torch.full((N, T, H, W, C), float("nan"), dtype=torch.float64)
    classes = plans.geom3_s2_dgrad_classes(N, T, H, W, Co)
    assert len(classes) == 8 and sorted(len(g.taps) for *_, g in classes) == [1, 2, 2, 2, 4, 4, 4, 8]
    for pt, ph, pw, gd in classes:
        strides, off = plans.s2_dgrad_out(T, H, W, C, pt, ph, pw)
        assert strides == (T * H * W * C, 2 * H * W * C, 2 * W * C, 2 * C, 1)
        assert off == ((pt * H + ph) * W + pw) * C
        ours[:, pt::2, ph::2, pw::2] = emulate_conv3d(gd, _to_cl(dy), pack3_t(w, gd.tapmap), C)
    assert torch.allclose(ours, _to_cl(gx), atol=1e-9)  # every voxel written once (no NaN left)
    g = plans.geom3_s2(N, T, H, W, C)
    part = emulate_wgrad3d(g, _to_cl(x), _to_cl(dy), Co)
    assert torch.allclose(reduce_tapmap(part, g.tapmap, w.shape), gw, atol=1e-9)


@pytest.mark.parametrize("shape", [(1, 3, 5, 7), (2, 2, 3, 4)])
def test_up_dgrad_64_taps_and_folded_wgrad_match_autograd(shape, f64):
    """Upsample (nearest x2 + 3x3x3 conv): the 64-tap data gradient over the 8 parity views of dy and the 8-phase folded
    weight gradient filling one partial buffer, against autograd of interpolate + conv3d."""
    torch.manual_seed(2)
    N, t_, h, w_ = shape
    C, Co = 8, 16
    x, w = torch.randn(N, C, t_, h, w_, dtype=torch.float64), torch.randn(Co, C, 3, 3, 3, dtype=torch.float64)
    dy = torch.randn(N, Co, 2 * t_, 2 * h, 2 * w_, dtype=torch.float64)
    gx, gw = _grads(lambda x_, w_p: F.conv3d(F.interpolate(x_, scale_factor=2.0, mode="nearest"), w_p, padding=1),
                    x, w, dy)
    gd = plans.geom3_up_dgrad(N, t_, h, w_, Co)
    assert len(gd.views) == 8 and len(gd.taps) == 64 and len(gd.taps) <= 64
    ours = emulate_conv3d(gd, _to_cl(dy), pack3_fold_t(w, gd.tapmask), C)
    assert torch.allclose(ours, _to_cl(gx), atol=1e-9)
    # weight gradient: phase p writes columns p*8*C .. of a [Cout][64 slots][C] partial
    part = torch.zeros(Co, 64, C, dtype=torch.float64)
    masks = []
    for pt in range(2):
        for ph in range(2):
            for pw in range(2):
                g = plans.geom3_up_fwd(N, t_, h, w_, C, pt, ph, pw)
                dv = plans.up3_dy_view(N, t_, h, w_, Co, pt, ph, pw)
                p = pt * 4 + ph * 2 + pw
                part[:, p * 8:(p + 1) * 8] = emulate_wgrad3d(g, _to_cl(x), _to_cl(dy), Co, dy_view=dv)
                masks += g.tapmask
    assert torch.allclose(reduce_fold(part, masks, w.shape), gw, atol=1e-9)


def test_1x1x1_plan_addresses_the_nthwc_tensor():
    """nin_shortcut / qkv / proj_out backward (Conv3dFn kind "p1"): the 2-D 1x1 dgrad plan and output strides on the
    [N][T*H][W] view address exactly the NTHWC tensor, and the 4-D view of the 5-D gradient buffer that the 2-D weight
    gradient writes is the parameter's gradient storage."""
    import ops

    N, T, H, W, Cp, Co = 2, 3, 4, 5, 16, 8
    gd = plans.geom_s1_dgrad(N, T * H, W, Co, 1)
    assert gd.taps == [(0, 0, 0)] and gd.tapmap == [0] and (gd.N, gd.Ho, gd.Wo) == (N, T * H, W)
    v = gd.views[0]
    dy = torch.arange(N * T * H * W * Co).view(N, T, H, W, Co)
    n, t, h, w = torch.meshgrid(*(torch.arange(e) for e in (N, T, H, W)), indexing="ij")
    off = v.offset + n * v.sn + (t * H + h) * v.sh + w * v.sw  # the view's voxel rows over the flattened grid
    assert torch.equal(dy.reshape(-1)[off.unsqueeze(-1) + torch.arange(Co)], dy)
    on, oh, ow, oc = plans.nhwc_strides(T * H, W, Cp)  # dgrad output strides over the flattened grid
    on3, ot3, oh3, ow3, oc3 = plans.nthwc_strides(T, H, W, Cp)
    assert torch.equal(n * on + (t * H + h) * oh + w * ow, n * on3 + t * ot3 + h * oh3 + w * ow3) and oc == oc3 == 1
    wt = torch.nn.Parameter(torch.zeros(Co, Cp, 1, 1, 1))
    gw = ops.grad_out(wt)
    g4 = gw.view(Co, Cp, 1, 1)
    assert gw.shape == wt.shape and g4.data_ptr() == gw.data_ptr() and g4.is_contiguous()
    g4[3, 5, 0, 0] = 7.0
    assert gw[3, 5, 0, 0, 0] == 7.0


def test_ksplit_counts_voxel_boxes():
    import ops

    g = plans.geom3_s1(1, 48, 256, 256, 64)
    ks = ops.choose_ksplit(g, 64)
    assert 1 <= ks <= 128
    small = plans.geom3_s1(1, 2, 4, 4, 64)  # one 64-voxel box: no split
    assert ops.choose_ksplit(small, 64) == 1


# ------------------------------------------------------------------------------------------------ C ABI
def test_struct_sizes_match_the_header():
    import native

    assert ctypes.sizeof(native.VqbConv3dDgradDesc) == 10 * 4 + 5 * 8 + 8 * 56 + 64 * 16
    assert ctypes.sizeof(native.VqbWgrad3dDesc) == 10 * 4 + 2 * 8 + 56 + 8 * 56 + 27 * 16
    # unchanged
    assert ctypes.sizeof(native.VqbConv3dDesc) == 10 * 4 + 5 * 8 + 8 * 56 + 27 * 16
    assert ctypes.sizeof(native.VqbWgradDesc) == 8 * 4 + 2 * 8 + 48 + 16 * 48 + 16 * 16
    assert ctypes.sizeof(native.VqbConvDesc) == 10 * 4 + 4 * 8 + 16 * 48 + 16 * 16


def test_struct_layouts_match_the_compiled_header(tmp_path):
    """sizeof and offsetof of every field of the new (and the pinned) descriptors, as a C compiler lays out
    include/vqb200.h, against the ctypes structs of native.py."""
    import shutil
    import subprocess

    import native

    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    structs = [native.VqbConv3dDgradDesc, native.VqbWgrad3dDesc, native.VqbConv3dDesc, native.VqbWgradDesc]
    lines = []
    for st in structs:
        n = st.__name__
        lines.append(f'printf("{n} sizeof %zu\\n", sizeof({n}));')
        for f, _ in st._fields_:
            lines.append(f'printf("{n} {f} %zu\\n", offsetof({n}, {f}));')
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "vqb200.h"\nint main(void) {\n' +
                   "\n".join(lines) + "\nreturn 0;\n}\n")
    exe = tmp_path / "probe"
    subprocess.run([cc, "-I", inc, str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    want = []
    for st in structs:
        want.append(f"{st.__name__} sizeof {ctypes.sizeof(st)}")
        want += [f"{st.__name__} {f} {getattr(st, f).offset}" for f, _ in st._fields_]
    assert [g for g in got if g] == want


@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    return native.load()


def _dgrad_desc(bad=None):
    d = plans.conv3d_dgrad_desc(plans.geom3_up_dgrad(1, 2, 4, 4, 16), 8, plans.nthwc_strides(2, 4, 4, 8))
    if bad == "flags":
        d.flags = 1
    elif bad == "taps":
        d.ntaps = 65
    elif bad == "view":
        d.taps[40].view = 8
    return d


def _wgrad_desc(bad=None):
    g = plans.geom3_s1(1, 2, 4, 4, 8)
    d = plans.wgrad3d_desc(g, 16, 1)
    if bad == "taps":
        d.ntaps = 28
    elif bad == "C":
        d.C = 12
    elif bad == "ksplit":
        d.ksplit = 0
    return d


def calls(p):
    return [
        ("vqb_conv3d_dgrad_gemm",
         lambda L: L.vqb_conv3d_dgrad_gemm(_dgrad_desc(), p, p, p, None),
         [lambda L: L.vqb_conv3d_dgrad_gemm(_dgrad_desc("flags"), p, p, p, None),
          lambda L: L.vqb_conv3d_dgrad_gemm(_dgrad_desc("taps"), p, p, p, None),
          lambda L: L.vqb_conv3d_dgrad_gemm(_dgrad_desc("view"), p, p, p, None),
          lambda L: L.vqb_conv3d_dgrad_gemm(_dgrad_desc(), p, None, p, None)]),
        ("vqb_wgrad3d_gemm",
         lambda L: L.vqb_wgrad3d_gemm(_wgrad_desc(), p, p, p, None),
         [lambda L: L.vqb_wgrad3d_gemm(_wgrad_desc("taps"), p, p, p, None),
          lambda L: L.vqb_wgrad3d_gemm(_wgrad_desc("C"), p, p, p, None),
          lambda L: L.vqb_wgrad3d_gemm(_wgrad_desc("ksplit"), p, p, p, None),
          lambda L: L.vqb_wgrad3d_gemm(_wgrad_desc(), p, p, p + 4, None)]),
        ("vqb_attn_bwd_hd",
         lambda L: L.vqb_attn_bwd_hd(p, p, p, p, p, p, 1, 64, 256, 32, None),
         [lambda L: L.vqb_attn_bwd_hd(p, p, p, p, p, p, 1, 64, 1024, 128, None),
          lambda L: L.vqb_attn_bwd_hd(p, p, p, p, p, p, 1, 64, 200, 32, None),
          lambda L: L.vqb_attn_bwd_hd(p, p, p, p, p, p + 8, 1, 64, 256, 32, None),
          lambda L: L.vqb_attn_bwd_hd(p, p, None, p, p, p, 1, 64, 256, 32, None)]),
        ("vqb_gauss_reparam_bwd",
         lambda L: L.vqb_gauss_reparam_bwd(p, p, p, p, 1, 4, 64, None),
         [lambda L: L.vqb_gauss_reparam_bwd(p, p, p, p, 1, 0, 64, None),
          lambda L: L.vqb_gauss_reparam_bwd(p, p, None, p, 1, 4, 64, None),
          lambda L: L.vqb_gauss_reparam_bwd(p, p, p, p + 2, 1, 4, 64, None)]),
    ]


def test_training_entry_points_are_declared_and_exported(lib):
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vqb200.h")).read()
    for name, _, _ in calls(0):
        assert f"int {name}(" in hdr, name
        assert hasattr(lib, name), name
    assert lib.vqb_version() >= 102


def test_training_entry_points_validate_and_fail_without_device(lib):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    for name, good, bads in calls(p):
        for i, bad in enumerate(bads):
            assert bad(lib) == EINVAL, (name, i)
        assert good(lib) == ENODEVICE, name
        assert b"sm_90" in lib.vqb_last_error(), name
    # the 27-tap forward descriptor still refuses 28 taps; the 64-tap one takes 64
    assert lib.vqb_conv3d_dgrad_gemm(_dgrad_desc(), p, p, p, None) == ENODEVICE


# ------------------------------------------------------------------------------------------------ module surface
def test_enable_training_sets_a_flag_and_keeps_the_state_dict():
    import tae

    torch.manual_seed(5)
    m = tae.TVAE(**SMALL.kwargs())
    torch.manual_seed(5)
    ref = tae.TVAE(**SMALL.kwargs())
    assert tae.enable_training(m) is m
    assert all(getattr(s, "_vqb_training", False) for s in m.modules())
    sd, sr = m.state_dict(), ref.state_dict()
    assert list(sd) == list(sr) and all(torch.equal(sd[k], sr[k]) for k in sd)
    tae.enable_training(m, False)
    assert not any(getattr(s, "_vqb_training", False) for s in m.modules())


def test_training_refusals_on_the_host():
    import tae

    x = torch.zeros(1, 3, 4, 16, 24)
    m = tae.TVAE(**SMALL.kwargs())
    with pytest.raises(RuntimeError, match="no_grad") as e:
        m(x)  # not opted in
    assert "enable_training" in str(e.value)
    tae.enable_training(m.bfloat16())
    with pytest.raises(RuntimeError, match="bfloat16.*inference-only"):
        m(x.bfloat16())
    with pytest.raises(RuntimeError, match="bfloat16"):
        m.decoder(torch.zeros(1, 4, 2, 8, 12, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="float16"):
        m.half()(x.half())
    z = torch.zeros(1, 8, 2, 8, 12, requires_grad=True)
    with pytest.raises(RuntimeError, match="no_grad"):
        tae.DiagonalGaussian()(z)
    with pytest.raises(RuntimeError, match="float32 latent"):
        tae.enable_training(tae.DiagonalGaussian())(z.detach().bfloat16().requires_grad_(True))


# ------------------------------------------------------------------------------------------------ reference gradients
def _probe(name, numel, i):  # as tools/make_tae_grad_golden.py
    g = torch.Generator().manual_seed(int.from_bytes(f"{name}/{i}".encode(), "little") % (2 ** 63))
    return torch.randn(numel, generator=g, dtype=torch.float64)


def _sample_idx(name, numel, k):
    g = torch.Generator().manual_seed(int.from_bytes(f"{name}/samples".encode(), "little") % (2 ** 63))
    return torch.randint(0, numel, (k,), generator=g)


def test_oracle_autograd_reproduces_reference_gradients():
    """oracle/tae_oracle.py under autograd against the unmodified reference tae.py (tests/golden/tae_grad_small.npz):
    the loss, the input gradient, and every parameter gradient's norm, probe projections and sampled values, in the
    reference's parameter order and shapes. The fixture's logvar lies on both sides of the clamp at -3."""
    import tae
    from helpers import golden, rel_l2, t
    from oracle import seeded

    gd = golden("tae_grad_small")
    assert 0.0 < float(gd["logvar_below"]) < 1.0
    m = tae.TVAE(**SMALL.kwargs())
    names = [n for n, _ in m.named_parameters()]
    assert names == [str(n) for n in gd["names"]]
    for i, (n, p) in enumerate(m.named_parameters()):
        assert list(p.shape) == [s for s in gd["shapes"][i] if s >= 0], n
    sd = {k: v.clone().requires_grad_(True) for k, v in seeded.fill_state_dict(m.state_dict(), "tae_small").items()}
    x = t(gd["x"]).clone().requires_grad_(True)
    decz, z = TO.forward(sd, x, t(gd["eps"]), SMALL)
    loss = ((decz - x) ** 2).mean() + 0.1 * (z ** 2).mean()
    loss.backward()
    assert abs(loss.item() - float(gd["loss"])) <= 1e-4 * abs(float(gd["loss"]))
    assert rel_l2(x.grad, gd["grad_x"]) < 1e-4
    norms = gd["grad_norms"]
    floor = 1e-6 * norms.max()  # mathematically-zero gradients (a bias in front of a GroupNorm) carry only noise
    for i, n in enumerate(names):
        v = sd[n].grad.double().reshape(-1)
        tol = 1e-4 * norms[i] + floor
        assert abs(v.norm().item() - norms[i]) <= tol, n
        proj = torch.stack([_probe(n, v.numel(), j) @ v for j in range(gd["grad_probes"].shape[1])])
        assert (proj - t(gd["grad_probes"][i])).abs().max().item() <= 4 * tol, n
        samp = v[_sample_idx(n, v.numel(), gd["grad_samples"].shape[1])]
        assert (samp - t(gd["grad_samples"][i])).abs().max().item() <= tol, n
