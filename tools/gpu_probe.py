"""GPU parity probe and micro-benchmarks for the wgmma conv / wgrad kernels and the other C ABI entry points (not a pytest file).

usage: python tools/gpu_probe.py <group>     groups: gemm conv conv2 wgrad elem
Each case prints one line: PASS/FAIL name max_abs_err rel_err; failures dump an error map.
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))

import torch
import torch.nn.functional as F

import native
import plans
from native import EPI_BIAS, EPI_MASK, EPI_RELU, EPI_RES

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
dev = "cuda"
L = native.load()


def report(name, got, ref, tol=2e-2):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    denom = ref.abs().max().item() + 1e-12
    mx = err.max().item()
    rel = mx / denom
    rel2 = ((got - ref).norm() / (ref.norm() + 1e-12)).item()
    ok = rel2 < tol and torch.isfinite(got).all().item()
    print(f"{'PASS' if ok else 'FAIL'} {name}: max_abs={mx:.4e} ref_max={denom:.3e} rel_l2={rel2:.3e}", flush=True)
    if not ok:
        e2 = err.reshape(-1, err.shape[-1])
        rows = e2.max(dim=1).values
        cols = e2.max(dim=0).values
        nr = min(rows.numel(), 128)
        print("  row-err(first %d, by 8):" % nr, [f"{rows[i:i+8].max().item():.2e}" for i in range(0, nr, 8)])
        nc = min(cols.numel(), 256)
        print("  col-err(by 16):", [f"{cols[i:i+16].max().item():.2e}" for i in range(0, nc, 16)])
        print("  got[0,:8]", got.reshape(-1, got.shape[-1])[0, :8].tolist())
        print("  ref[0,:8]", ref.reshape(-1, ref.shape[-1])[0, :8].tolist())
    return ok


def pack_torch(w, tapmap, transpose, Kpad):
    """w: [Cout,Cin,KH,KW] fp32 -> bf16 [R][slots][Kpad]"""
    Cout, Cin = w.shape[:2]
    wt = w.reshape(Cout, Cin, -1)[:, :, tapmap]  # [Cout,Cin,slots]
    if transpose:
        m = wt.permute(1, 2, 0)  # [Cin, slots, Cout]
    else:
        m = wt.permute(0, 2, 1)  # [Cout, slots, Cin]
    out = torch.zeros(m.shape[0], m.shape[1], Kpad, device=w.device, dtype=torch.bfloat16)
    out[:, :, : m.shape[2]] = m.to(torch.bfloat16)
    return out.contiguous()


def run_conv(g, x, wp, Cout, bias=None, res=None, mask=None, relu=False, out=None, out_strides=None, out_f32=False):
    flags = 0
    if bias is not None:
        flags |= EPI_BIAS
    if res is not None:
        flags |= EPI_RES
    if mask is not None:
        flags |= EPI_MASK
    if relu:
        flags |= EPI_RELU
    Cs = plans.cpad(Cout)
    if out is None:
        out = torch.zeros(g.N, g.Ho, g.Wo, Cs, device=dev, dtype=torch.bfloat16)
        out_strides = plans.nhwc_strides(g.Ho, g.Wo, Cs)
    d = plans.conv_desc(g, Cout, out_strides, flags, out_f32)
    rc = L.vqb_conv_gemm(d, native.ptr(x), native.ptr(wp), native.ptr(bias), native.ptr(res), native.ptr(mask),
                         native.ptr(out), 0, native.stream_ptr())
    native.check(rc, "conv_gemm")
    torch.cuda.synchronize()
    return out


def rnd(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale)


def case_gemm(M, K, Nn, seed=0):
    torch.manual_seed(seed)
    a = rnd(1, 1, M, K).to(torch.bfloat16)
    w = rnd(Nn, K, 1, 1, scale=K ** -0.5)
    g = plans.geom_s1(1, 1, M, K, 1)
    wp = pack_torch(w, g.tapmap, False, K)
    out = run_conv(g, a, wp, Nn)
    ref = a.float().reshape(M, K) @ wp.float().reshape(Nn, K).t()
    return report(f"gemm M={M} K={K} N={Nn}", out.reshape(M, -1)[:, :Nn], ref)


def case_conv(N, H, W, Cin, Cout, k, seed=0, bias=False, res=False, relu=False, mask=False, nchw_f32=False):
    torch.manual_seed(seed)
    Cp = plans.cpad(Cin)
    x = torch.zeros(N, H, W, Cp, device=dev, dtype=torch.bfloat16)
    x[..., :Cin] = rnd(N, H, W, Cin).to(torch.bfloat16)
    w = rnd(Cout, Cin, k, k, scale=(Cin * k * k) ** -0.5)
    g = plans.geom_s1(N, H, W, Cp, k)
    wp = pack_torch(w, g.tapmap, False, Cp)
    b = rnd(Cout) if bias else None
    Cs = plans.cpad(Cout)
    r = rnd(N, H, W, Cs).to(torch.bfloat16) if res else None
    mk = rnd(N, H, W, Cs).to(torch.bfloat16) if mask else None
    ref = F.conv2d(x[..., :Cin].float().permute(0, 3, 1, 2), wp.float().reshape(Cout, k * k, Cp)[:, :, :Cin]
                   .permute(0, 2, 1).reshape(Cout, Cin, k, k), b, padding=(k - 1) // 2)
    if res:
        ref = ref + r[..., :Cout].float().permute(0, 3, 1, 2)
    if relu:
        ref = ref.relu()
    if mask:
        ref = ref * (mk[..., :Cout].float().permute(0, 3, 1, 2) > 0)
    if nchw_f32:
        out = torch.zeros(N, Cout, H, W, device=dev, dtype=torch.float32)
        run_conv(g, x, wp, Cout, b, r, mk, relu, out=out, out_strides=plans.nchw_strides(Cout, H, W), out_f32=True)
        got = out
    else:
        out = run_conv(g, x, wp, Cout, b, r, mk, relu)
        got = out[..., :Cout].permute(0, 3, 1, 2)
    tag = f"conv{k}x{k} N={N} {H}x{W} {Cin}->{Cout}" + (" +bias" if bias else "") + (" +res" if res else "") + \
        (" +relu" if relu else "") + (" +mask" if mask else "") + (" nchw_f32" if nchw_f32 else "")
    return report(tag, got.permute(0, 2, 3, 1), ref.permute(0, 2, 3, 1))


def case_conv_s2(N, H, W, C, Cout, seed=0):
    torch.manual_seed(seed)
    x = rnd(N, H, W, C).to(torch.bfloat16)
    w = rnd(Cout, C, 3, 3, scale=(C * 9) ** -0.5)
    g = plans.geom_s2(N, H, W, C)
    wp = pack_torch(w, g.tapmap, False, C)
    out = run_conv(g, x, wp, Cout)
    xp = F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1))
    ref = F.conv2d(xp, w.to(torch.bfloat16).float(), stride=2)
    return report(f"conv3x3s2 N={N} {H}x{W} {C}->{Cout}", out.float(), ref.permute(0, 2, 3, 1))


def case_dgrad_s1(N, H, W, Cin, Cout, k, seed=0):
    """dx = conv_transpose(dy, w): run as conv over dy with transposed/rotated packed weights."""
    torch.manual_seed(seed)
    Cop = plans.cpad(Cout)
    dy = torch.zeros(N, H, W, Cop, device=dev, dtype=torch.bfloat16)
    dy[..., :Cout] = rnd(N, H, W, Cout).to(torch.bfloat16)
    w = rnd(Cout, Cin, k, k, scale=(Cout * k * k) ** -0.5)
    g = plans.geom_s1_dgrad(N, H, W, Cop, k)
    wp = pack_torch(w, g.tapmap, True, Cop)
    out = run_conv(g, dy, wp, Cin)
    ref = F.conv_transpose2d(dy[..., :Cout].float().permute(0, 3, 1, 2), w.to(torch.bfloat16).float(),
                             padding=(k - 1) // 2)
    return report(f"dgrad{k}x{k} N={N} {H}x{W} Cin={Cin} Cout={Cout}", out[..., :Cin].float(),
                  ref.permute(0, 2, 3, 1))


def case_dgrad_s2(N, H, W, C, Cout, seed=0):
    torch.manual_seed(seed)
    Ho, Wo = H // 2, W // 2
    dy = rnd(N, Ho, Wo, Cout).to(torch.bfloat16)
    w = rnd(Cout, C, 3, 3, scale=(Cout * 9) ** -0.5)
    dx = torch.zeros(N, H, W, C, device=dev, dtype=torch.bfloat16)
    for ph, pw, g in plans.geom_s2_dgrad_classes(N, H, W, Cout):
        wp = pack_torch(w, g.tapmap, True, Cout)
        sub = dx[:, ph::2, pw::2, :]
        strides = (H * W * C, 2 * W * C, 2 * C, 1)
        d = plans.conv_desc(g, C, strides, 0, False)
        base = dx.data_ptr() + (ph * W + pw) * C * 2
        rc = L.vqb_conv_gemm(d, native.ptr(dy), native.ptr(wp), 0, 0, 0, base, 0, native.stream_ptr())
        native.check(rc, "conv_gemm dgrad s2")
    torch.cuda.synchronize()
    x = torch.zeros(N, C, H, W, device=dev, requires_grad=True)
    y = F.conv2d(F.pad(x, (0, 1, 0, 1)), w.to(torch.bfloat16).float(), stride=2)
    (ref,) = torch.autograd.grad(y, x, dy.float().permute(0, 3, 1, 2))
    return report(f"dgrad3x3s2 N={N} {H}x{W} {C}<-{Cout}", dx.float(), ref.permute(0, 2, 3, 1))


def case_wgrad(N, H, W, Cin, Cout, k, ksplit, stride2=False, seed=0):
    torch.manual_seed(seed)
    Cp, Cop = plans.cpad(Cin), plans.cpad(Cout)
    x = torch.zeros(N, H, W, Cp, device=dev, dtype=torch.bfloat16)
    x[..., :Cin] = rnd(N, H, W, Cin).to(torch.bfloat16)
    g = plans.geom_s2(N, H, W, Cp) if stride2 else plans.geom_s1(N, H, W, Cp, k)
    dy = torch.zeros(N, g.Ho, g.Wo, Cop, device=dev, dtype=torch.bfloat16)
    dy[..., :Cout] = rnd(N, g.Ho, g.Wo, Cout).to(torch.bfloat16)
    d = plans.wgrad_desc(g, Cop, ksplit)
    cols = L.vqb_wgrad_cols(len(g.taps), Cp)
    partial = torch.full((ksplit, Cop, cols), float("nan"), device=dev, dtype=torch.float32)
    rc = L.vqb_wgrad_gemm(d, native.ptr(dy), native.ptr(x), native.ptr(partial), native.stream_ptr())
    native.check(rc, "wgrad_gemm")
    T = k * k
    grad = torch.zeros(Cout, Cin, k, k, device=dev, dtype=torch.float32)
    tapmap = torch.tensor(g.tapmap, device=dev, dtype=torch.int32)
    rc = L.vqb_wgrad_reduce(native.ptr(partial), native.ptr(grad), ksplit, Cout, Cop, Cin, T, len(g.taps),
                            cols // len(g.taps), native.ptr(tapmap), 0, native.stream_ptr())
    native.check(rc, "wgrad_reduce")
    torch.cuda.synchronize()
    wref = torch.zeros(Cout, Cin, k, k, device=dev, requires_grad=True)
    xin = x[..., :Cin].float().permute(0, 3, 1, 2)
    if stride2:
        y = F.conv2d(F.pad(xin, (0, 1, 0, 1)), wref, stride=2)
    else:
        y = F.conv2d(xin, wref, padding=(k - 1) // 2)
    (ref,) = torch.autograd.grad(y, wref, dy[..., :Cout].float().permute(0, 3, 1, 2))
    C64 = cols // len(g.taps)
    got_p = partial.sum(0)[:Cout].reshape(Cout, len(g.taps), C64)[:, :, :Cin]  # [Cout, slot, Cin]
    ref_p = ref.reshape(Cout, Cin, T).permute(0, 2, 1)
    ok = report(f"wgrad{k}x{k}{'s2' if stride2 else ''} N={N} {H}x{W} {Cin}->{Cout} ksplit={ksplit} (partial)",
                got_p.reshape(Cout, -1), ref_p.reshape(Cout, -1), tol=1e-2)
    if rc == 0:
        ok &= report("   + reduce->OIHW", grad.reshape(Cout, -1), ref.reshape(Cout, -1), tol=1e-2)
    return ok


def bench_conv(N, H, W, Cin, Cout, k, iters=20, res=False, cudnn=True):
    torch.manual_seed(0)
    x = rnd(N, H, W, Cin).to(torch.bfloat16)
    w = rnd(Cout, Cin, k, k, scale=(Cin * k * k) ** -0.5)
    g = plans.geom_s1(N, H, W, Cin, k)
    wp = pack_torch(w, g.tapmap, False, Cin)
    out = torch.zeros(N, H, W, Cout, device=dev, dtype=torch.bfloat16)
    d = plans.conv_desc(g, Cout, plans.nhwc_strides(H, W, Cout), native.EPI_RES if res else 0, False)
    r = rnd(N, H, W, Cout).to(torch.bfloat16) if res else None
    args = (d, native.ptr(x), native.ptr(wp), 0, native.ptr(r), 0, native.ptr(out), 0, native.stream_ptr())
    for _ in range(3):
        native.check(L.vqb_conv_gemm(*args))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        L.vqb_conv_gemm(*args)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * N * H * W * Cout * Cin * k * k
    if not cudnn or res:
        print(f"BENCH conv{k}x{k} N={N} {H}x{W} {Cin}->{Cout}{' +res' if res else ''}: ours {ms:.3f} ms = "
              f"{fl / ms / 1e9:.1f} TFLOP/s", flush=True)
        return
    # cudnn bf16 reference timing
    xc = x.permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    wc = w.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    for _ in range(3):
        F.conv2d(xc, wc, padding=(k - 1) // 2)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        F.conv2d(xc, wc, padding=(k - 1) // 2)
    e1.record()
    torch.cuda.synchronize()
    ms_ref = e0.elapsed_time(e1) / iters
    print(f"BENCH conv{k}x{k} N={N} {H}x{W} {Cin}->{Cout}: ours {ms:.3f} ms = {fl / ms / 1e9:.1f} TFLOP/s | "
          f"cudnn bf16 {ms_ref:.3f} ms = {fl / ms_ref / 1e9:.1f} TFLOP/s", flush=True)


def bench_wgrad(N, H, W, Cin, Cout, k, ksplit, iters=10):
    torch.manual_seed(0)
    x = rnd(N, H, W, Cin).to(torch.bfloat16)
    dy = rnd(N, H, W, Cout).to(torch.bfloat16)
    g = plans.geom_s1(N, H, W, Cin, k)
    d = plans.wgrad_desc(g, Cout, ksplit)
    cols = L.vqb_wgrad_cols(len(g.taps), Cin)
    partial = torch.zeros(ksplit, Cout, cols, device=dev, dtype=torch.float32)
    args = (d, native.ptr(dy), native.ptr(x), native.ptr(partial), native.stream_ptr())
    for _ in range(2):
        native.check(L.vqb_wgrad_gemm(*args))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        L.vqb_wgrad_gemm(*args)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * N * H * W * Cout * Cin * k * k
    print(f"BENCH wgrad{k}x{k} N={N} {H}x{W} {Cin}->{Cout} ksplit={ksplit}: {ms:.3f} ms = {fl / ms / 1e9:.1f} TFLOP/s",
          flush=True)


def group_elem():
    ok = True
    torch.manual_seed(0)
    # pack_weights vs torch
    for (Cout, Cin, k, tr) in [(64, 48, 3, 0), (64, 48, 3, 1), (5, 128, 1, 0), (128, 3, 3, 1)]:
        w = rnd(Cout, Cin, k, k)
        tapmap = list(range(k * k))[::-1] if tr else list(range(k * k))
        Kpad = plans.cpad(Cout if tr else Cin)
        R = Cin if tr else Cout
        out = torch.zeros(R, k * k, Kpad, device=dev, dtype=torch.bfloat16)
        tm = torch.tensor(tapmap, device=dev, dtype=torch.int32)
        native.check(L.vqb_pack_weights(native.ptr(w), native.ptr(out), Cout, Cin, k * k, k * k, native.ptr(tm), tr,
                                        Kpad, native.stream_ptr()))
        torch.cuda.synchronize()
        ok &= report(f"pack_weights {Cout}x{Cin}x{k} tr={tr}", out.reshape(R, -1), pack_torch(w, tapmap, bool(tr), Kpad).reshape(R, -1), tol=1e-6)
    # layout conversion
    x = rnd(2, 3, 24, 40)
    shift = torch.tensor([-0.03, -0.088, -0.188], device=dev)
    iscale = 1.0 / torch.tensor([0.458, 0.448, 0.45], device=dev)
    y = torch.full((2, 24, 40, 8), 7.0, device=dev, dtype=torch.bfloat16)
    native.check(L.vqb_nchw_to_nhwc(native.ptr(x), native.ptr(y), 2, 3, 24, 40, 8, native.ptr(shift), native.ptr(iscale), native.stream_ptr()))
    torch.cuda.synchronize()
    ref = torch.zeros(2, 24, 40, 8, device=dev)
    ref[..., :3] = ((x - shift[None, :, None, None]) * iscale[None, :, None, None]).permute(0, 2, 3, 1)
    ok &= report("nchw_to_nhwc scaled", y, ref, tol=1e-2)
    gx = torch.zeros(2, 3, 24, 40, device=dev)
    native.check(L.vqb_nhwc_to_nchw(native.ptr(y), native.ptr(gx), 2, 3, 24, 40, 8, native.ptr(iscale), native.stream_ptr()))
    torch.cuda.synchronize()
    ok &= report("nhwc_to_nchw scaled", gx.permute(0, 2, 3, 1), y[..., :3].float() * iscale, tol=1e-6)
    # GroupNorm + SiLU fwd/bwd
    for (N, H, W, Cc, silu) in [(2, 16, 16, 128, 1), (3, 8, 8, 32, 1), (1, 64, 64, 256, 0), (2, 32, 32, 512, 1), (2, 10, 6, 64, 1)]:
        xx = (rnd(N, H, W, Cc) * 2 + 0.5).to(torch.bfloat16)
        gamma = rnd(Cc) * 0.5 + 1
        beta = rnd(Cc) * 0.2
        yy = torch.zeros_like(xx)
        mr = torch.zeros(N, 32, 2, device=dev)
        ws = torch.zeros(N * Cc * 2, device=dev, dtype=torch.float64)
        native.check(L.vqb_gn_silu_fwd(native.ptr(xx), native.ptr(yy), native.ptr(gamma), native.ptr(beta), native.ptr(mr),
                                       native.ptr(ws), N, H * W, Cc, 32, 1e-6, silu, native.stream_ptr()))
        torch.cuda.synchronize()
        xr = xx.float().permute(0, 3, 1, 2).requires_grad_(True)
        gr = gamma.clone().requires_grad_(True)
        br = beta.clone().requires_grad_(True)
        yr = F.group_norm(xr, 32, gr, br, 1e-6)
        if silu:
            yr = yr * torch.sigmoid(yr)
        ok &= report(f"gn_silu_fwd N={N} {H}x{W} C={Cc} silu={silu}", yy, yr.permute(0, 2, 3, 1), tol=1e-2)
        dy = rnd(N, H, W, Cc).to(torch.bfloat16)
        addt = rnd(N, H, W, Cc).to(torch.bfloat16)
        dx = torch.zeros_like(xx)
        dg = torch.zeros(Cc, device=dev)
        db = torch.zeros(Cc, device=dev)
        ws2 = torch.zeros(N * Cc * 2 + N * 32 * 2, device=dev)
        csum = torch.full((Cc,), 7.0, device=dev)
        native.check(L.vqb_gn_silu_bwd(native.ptr(xx), native.ptr(dy), native.ptr(addt), native.ptr(dx), native.ptr(gamma),
                                       native.ptr(beta), native.ptr(mr), native.ptr(dg), native.ptr(db), native.ptr(ws2),
                                       N, H * W, Cc, 32, silu, native.ptr(csum), native.stream_ptr()))
        torch.cuda.synchronize()
        ok &= report("   bwd colsum(dx)", csum[None], dx.float().sum((0, 1, 2))[None], tol=1e-3)
        gxr, ggr, gbr = torch.autograd.grad(yr, (xr, gr, br), dy.float().permute(0, 3, 1, 2))
        ok &= report("   bwd dx(+add)", dx, gxr.permute(0, 2, 3, 1) + addt.float(), tol=1e-2)
        ok &= report("   bwd dgamma", dg[None], ggr[None], tol=1e-2)
        ok &= report("   bwd dbeta", db[None], gbr[None], tol=1e-2)
    # colsum
    xc = rnd(5000, 128).to(torch.bfloat16)
    oc = torch.zeros(128, device=dev)
    native.check(L.vqb_colsum(native.ptr(xc), native.ptr(oc), 5000, 128, native.stream_ptr()))
    torch.cuda.synchronize()
    ok &= report("colsum", oc[None], xc.float().sum(0)[None], tol=1e-3)
    return ok


def group_lpips():
    ok = True
    torch.manual_seed(0)
    # max-pool fwd / bwd (ReLU-gated, first-max tie rule)
    for (N, H, W, Cc) in [(2, 16, 16, 64), (1, 8, 24, 128)]:
        x = rnd(N, H, W, Cc).relu().to(torch.bfloat16)
        x[0, 0:2, 0:2, :] = 1.0  # ties
        y = torch.zeros(N, H // 2, W // 2, Cc, device=dev, dtype=torch.bfloat16)
        native.check(L.vqb_maxpool2_fwd(native.ptr(x), native.ptr(y), N, H // 2, W // 2, Cc, native.stream_ptr()))
        xr = x.float().permute(0, 3, 1, 2).requires_grad_(True)
        yr = F.max_pool2d(xr, 2)
        torch.cuda.synchronize()
        ok &= report(f"maxpool2 fwd {N}x{H}x{W}x{Cc}", y, yr.permute(0, 2, 3, 1), tol=1e-6)
        dy = rnd(N, H // 2, W // 2, Cc).to(torch.bfloat16)
        dx = torch.zeros_like(x)
        native.check(L.vqb_maxpool2_bwd(native.ptr(x), native.ptr(dy), 0, native.ptr(dx), N, H // 2, W // 2, Cc, 1,
                                        native.stream_ptr()))
        torch.cuda.synchronize()
        (gref,) = torch.autograd.grad(yr, xr, dy.float().permute(0, 3, 1, 2))
        gref = gref * (xr > 0)
        ok &= report("   bwd (relu gated)", dx, gref.permute(0, 2, 3, 1), tol=1e-6)
    # LPIPS tail
    for (N, H, W, Cc) in [(2, 16, 16, 64), (2, 8, 8, 128), (3, 4, 4, 256), (2, 4, 4, 512), (1, 32, 32, 64)]:
        f0 = rnd(N, H, W, Cc).relu().to(torch.bfloat16)
        f1 = rnd(N, H, W, Cc).relu().to(torch.bfloat16)
        w = torch.rand(Cc, device=dev) / Cc
        out = torch.zeros(N, device=dev)
        native.check(L.vqb_lpips_tail_fwd(native.ptr(f0), native.ptr(f1), native.ptr(w), native.ptr(out), N, H * W, Cc,
                                          native.stream_ptr()))
        a = f0.float().permute(0, 3, 1, 2).requires_grad_(True)
        b = f1.float().permute(0, 3, 1, 2)

        def nrm(t_):
            return t_ / (torch.sqrt(torch.sum(t_ ** 2, dim=1, keepdim=True)) + 1e-10)

        ref = (F.conv2d((nrm(a) - nrm(b)) ** 2, w.view(1, Cc, 1, 1))).mean([2, 3]).reshape(N)
        torch.cuda.synchronize()
        ok &= report(f"lpips_tail fwd {N}x{H}x{W}x{Cc}", out[None], ref[None], tol=1e-4)
        g = torch.rand(N, device=dev) + 0.5
        df0 = torch.zeros_like(f0)
        native.check(L.vqb_lpips_tail_bwd(native.ptr(f0), native.ptr(f1), native.ptr(w), native.ptr(g), native.ptr(df0),
                                          N, H * W, Cc, native.stream_ptr()))
        torch.cuda.synchronize()
        (gref,) = torch.autograd.grad(ref, a, g)
        gref = gref * (a > 0)
        ok &= report("   bwd (relu gated)", df0, gref.permute(0, 2, 3, 1), tol=1e-2)
    return ok


def group_up():
    """nearest-2x upsample + conv3x3 folded into 4 phase convs (ops.UpConvFn) vs F.interpolate + F.conv2d autograd."""
    import ops
    ok = True
    torch.manual_seed(0)
    for (N, h, w, Ci, Co) in [(2, 16, 16, 128, 128), (1, 32, 32, 256, 256), (2, 8, 8, 64, 64), (1, 12, 20, 64, 128)]:
        x = rnd(N, h, w, Ci).to(torch.bfloat16).requires_grad_(True)
        wt = (rnd(Co, Ci, 3, 3) * (Ci * 9) ** -0.5).requires_grad_(True)
        b = rnd(Co).requires_grad_(True)
        cache = ops.PackedCache()
        y = ops.upsample_conv(x, wt, b, cache)
        gy = rnd(N, 2 * h, 2 * w, Co).to(torch.bfloat16)
        y.backward(gy)
        xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
        wr = wt.detach().clone().requires_grad_(True)
        br = b.detach().clone().requires_grad_(True)
        yr = F.conv2d(F.interpolate(xr, scale_factor=2.0, mode="nearest"), wr, br, padding=1)
        yr.backward(gy.float().permute(0, 3, 1, 2))
        tag = f"upconv N={N} {h}x{w} {Ci}->{Co}"
        ok &= report(tag + " fwd", y, yr.permute(0, 2, 3, 1), tol=1e-2)  # folded weights are rounded after the fp32 sum
        ok &= report("   dx", x.grad, xr.grad.permute(0, 2, 3, 1), tol=1e-2)
        ok &= report("   dW", wt.grad.reshape(Co, -1), wr.grad.reshape(Co, -1), tol=1e-2)
        ok &= report("   db", b.grad[None], br.grad[None], tol=1e-2)
    return ok


def group_stats():
    """GroupNorm statistics accumulated by the conv epilogue (VQB_EPI_STATS) + vqb_gn_silu_fwd_pre vs torch."""
    import ops
    ok = True
    torch.manual_seed(0)
    for (N, H, W, Ci, Co, res) in [(2, 32, 32, 64, 128, False), (2, 64, 64, 128, 128, True), (1, 32, 32, 512, 512, True),
                                   (3, 16, 16, 64, 64, False)]:
        x = rnd(N, H, W, Ci).to(torch.bfloat16)
        wt = rnd(Co, Ci, 3, 3) * (Ci * 9) ** -0.5
        b = rnd(Co)
        r = rnd(N, H, W, Co).to(torch.bfloat16) if res else None
        cache = ops.PackedCache()
        out, st = ops.conv(x, wt, b, cache, "s1", residual=r, want_stats=True)
        torch.cuda.synchronize()
        tag = f"conv+stats N={N} {H}x{W} {Ci}->{Co} res={res}"
        if st is None:
            print("SKIP (stats unsupported)", tag)
            continue
        of = out.float()
        ref = torch.stack([of.sum((1, 2)), (of * of).sum((1, 2))], dim=-1)  # [N, C, 2]
        ok &= report(tag + " sums", st.reshape(N, -1), ref.reshape(N, -1), tol=1e-4)
        gamma, beta = rnd(Co) * 0.5 + 1, rnd(Co) * 0.2
        y = ops.group_norm_silu(out, gamma, beta, 32, 1e-6, True, chsums=st)
        yr = F.group_norm(of.permute(0, 3, 1, 2), 32, gamma, beta, 1e-6)
        yr = (yr * torch.sigmoid(yr)).permute(0, 2, 3, 1)
        ok &= report("   gn_silu via conv-epilogue statistics", y, yr, tol=1e-2)
    # folded upsample conv accumulates the four phase launches into one statistics tensor
    x = rnd(2, 16, 16, 128).to(torch.bfloat16)
    wt = rnd(128, 128, 3, 3) * (128 * 9) ** -0.5
    out, st = ops.upsample_conv(x, wt, rnd(128), ops.PackedCache(), want_stats=True)
    torch.cuda.synchronize()
    if st is not None:
        of = out.float()
        ref = torch.stack([of.sum((1, 2)), (of * of).sum((1, 2))], dim=-1)
        ok &= report("upconv+stats sums", st.reshape(2, -1), ref.reshape(2, -1), tol=1e-4)
    else:
        print("SKIP upconv stats unsupported")
    return ok


def group_fat():
    """first-layer fat-pixel conv (3 taps of 24 over a zero-framed 8-channel image) vs the ordinary 9-tap path and torch."""
    import ops
    ok = True
    print("fat_conv_enabled:", ops.fat_conv_enabled())
    if not ops.fat_conv_enabled():
        return True  # the self-check disabled the path; the ordinary kernels are used
    torch.manual_seed(0)
    for (N, H, W, Co) in [(2, 32, 32, 64), (1, 64, 48, 128), (3, 20, 20, 64)]:
        x = (torch.rand(N, 3, H, W, device=dev) - 0.5).requires_grad_(True)
        wt = ((torch.rand(Co, 3, 3, 3, device=dev) - 0.5) * 0.5).requires_grad_(True)
        b = rnd(Co).requires_grad_(True)
        y = ops.conv(ops.to_nhwc(x, None, None, True), wt, b, ops.PackedCache(), "fat3")
        gy = rnd(N, H, W, Co).to(torch.bfloat16)
        y.backward(gy)
        xr = x.detach().to(torch.bfloat16).float().requires_grad_(True)
        wr = wt.detach().clone().requires_grad_(True)
        br = b.detach().clone().requires_grad_(True)
        yr = F.conv2d(xr, wr, br, padding=1)
        yr.backward(gy.float().permute(0, 3, 1, 2))
        tag = f"fat3 N={N} {H}x{W} 3->{Co}"
        ok &= report(tag + " fwd", y, yr.permute(0, 2, 3, 1), tol=1e-2)
        ok &= report("   dx", x.grad.permute(0, 2, 3, 1), xr.grad.permute(0, 2, 3, 1), tol=1e-2)
        ok &= report("   dW", wt.grad.reshape(Co, -1), wr.grad.reshape(Co, -1), tol=1e-2)
        ok &= report("   db", b.grad[None], br.grad[None], tol=1e-2)
    # tiny-Cout conv with NCHW fp32 output (decoder conv_out): framed dy -> fat data gradient
    x = rnd(2, 32, 32, 128).to(torch.bfloat16).requires_grad_(True)
    wt = (rnd(3, 128, 3, 3) * (128 * 9) ** -0.5).requires_grad_(True)
    b = rnd(3).requires_grad_(True)
    y = ops.conv(x, wt, b, ops.PackedCache(), "s1", nchw_out=True)
    gy = rnd(2, 3, 32, 32)
    y.backward(gy)
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = wt.detach().clone().requires_grad_(True)
    br = b.detach().clone().requires_grad_(True)
    yr = F.conv2d(xr, wr, br, padding=1)
    yr.backward(gy)
    ok &= report("conv_out 128->3 nchw fwd", y.permute(0, 2, 3, 1), yr.permute(0, 2, 3, 1), tol=1e-2)
    ok &= report("   dx (fat dgrad over framed dy)", x.grad, xr.grad.permute(0, 2, 3, 1), tol=1e-2)
    ok &= report("   dW", wt.grad.reshape(3, -1), wr.grad.reshape(3, -1), tol=1e-2)
    ok &= report("   db", b.grad[None], br.grad[None], tol=1e-2)
    return ok


def group_gemm():
    ok = True
    ok &= case_gemm(128, 64, 16)
    ok &= case_gemm(128, 64, 64)
    ok &= case_gemm(256, 128, 128)
    ok &= case_gemm(1024, 512, 256)
    ok &= case_gemm(4096, 256, 512)
    ok &= case_gemm(200, 64, 40)
    return ok


def group_conv():
    ok = True
    ok &= case_conv(2, 16, 16, 64, 64, 1)
    ok &= case_conv(2, 16, 16, 64, 64, 3)
    ok &= case_conv(2, 32, 32, 128, 128, 3, bias=True)
    ok &= case_conv(2, 32, 32, 512, 512, 3, bias=True, res=True)
    ok &= case_conv(1, 256, 256, 128, 128, 3)
    ok &= case_conv(4, 8, 8, 64, 128, 3, relu=True, bias=True)
    ok &= case_conv(3, 4, 4, 64, 64, 3)
    ok &= case_conv(2, 20, 20, 64, 64, 3, bias=True)
    ok &= case_conv(1, 24, 40, 128, 64, 3)
    # residual / mask operands arrive through TMA-prefetched tiles: ragged tiles, partial channel groups, many tiles per CTA
    ok &= case_conv(2, 20, 20, 64, 96, 3, bias=True, res=True)
    ok &= case_conv(3, 24, 40, 128, 32, 3, res=True, relu=True)
    ok &= case_conv(8, 128, 128, 128, 128, 3, bias=True, res=True)
    ok &= case_conv(8, 64, 64, 256, 256, 3, bias=True, res=True)
    ok &= case_conv(8, 64, 64, 128, 320, 1, res=True)
    ok &= case_conv(8, 64, 64, 128, 128, 3, mask=True)
    ok &= case_conv(2, 20, 20, 64, 96, 3, bias=True, res=True, mask=True)
    ok &= case_conv(5, 12, 12, 64, 64, 3, mask=True, relu=True)
    # Cout = 128, H >= 32: ragged tiles, every epilogue operand
    ok &= case_conv(3, 40, 20, 128, 128, 3, bias=True, res=True, relu=True)
    ok &= case_conv(2, 48, 24, 64, 128, 3, bias=True, mask=True)
    ok &= case_conv(9, 64, 64, 256, 128, 3, bias=True)
    ok &= case_conv(4, 128, 128, 128, 128, 3, res=True)
    ok &= case_conv(2, 32, 32, 128, 128, 3, bias=True)
    return ok


def group_conv2():
    ok = True
    ok &= case_conv(2, 32, 32, 16, 512, 3, bias=True)
    ok &= case_conv(2, 32, 32, 32, 64, 3)
    ok &= case_conv(2, 32, 32, 3, 128, 3, bias=True)
    ok &= case_conv(2, 32, 32, 512, 16, 3, bias=True, nchw_f32=True)
    ok &= case_conv(2, 64, 64, 128, 3, 3, bias=True, nchw_f32=True)
    ok &= case_conv(2, 32, 32, 128, 128, 3, mask=True)
    ok &= case_conv(2, 32, 32, 128, 3, 3)
    ok &= case_conv_s2(2, 32, 32, 128, 128)
    ok &= case_conv_s2(1, 64, 64, 256, 256)
    ok &= case_dgrad_s1(2, 32, 32, 128, 256, 3)
    ok &= case_dgrad_s1(2, 16, 16, 64, 64, 1)
    ok &= case_dgrad_s1(2, 32, 32, 3, 64, 3)
    ok &= case_dgrad_s2(2, 32, 32, 128, 128)
    return ok


def group_wgrad():
    ok = True
    ok &= case_wgrad(2, 16, 16, 64, 64, 1, 1)
    ok &= case_wgrad(2, 16, 16, 64, 64, 3, 1)
    ok &= case_wgrad(2, 32, 32, 128, 128, 3, 4)
    ok &= case_wgrad(2, 32, 32, 128, 256, 3, 2)
    ok &= case_wgrad(2, 16, 16, 512, 512, 3, 3)
    ok &= case_wgrad(1, 64, 64, 256, 128, 1, 8)
    ok &= case_wgrad(2, 20, 20, 64, 64, 3, 2)
    ok &= case_wgrad(4, 4, 4, 64, 64, 3, 1)
    ok &= case_wgrad(2, 32, 32, 16, 512, 3, 2)
    ok &= case_wgrad(2, 32, 32, 128, 128, 3, 2, stride2=True)
    return ok


def group_convbench():
    """3x3 convs at the FLUX-config shapes, against cuDNN, and with a residual epilogue operand"""
    for (N, H, W, Ci, Co) in [(32, 256, 256, 128, 128), (32, 128, 128, 256, 256), (32, 64, 64, 512, 512),
                              (32, 32, 32, 512, 512), (32, 16, 16, 512, 512), (32, 128, 128, 128, 256),
                              (32, 256, 256, 64, 64)]:
        bench_conv(N, H, W, Ci, Co, 3, cudnn=True)
        bench_conv(N, H, W, Ci, Co, 3, res=True)
    return True


def group_wgbench():
    """weight-gradient GEMM: split-K sweep per shape"""
    import ops
    for (N, H, W, Ci, Co) in [(32, 32, 32, 512, 512), (32, 256, 256, 128, 128), (32, 64, 64, 512, 512),
                              (32, 128, 128, 256, 256)]:
        g = plans.geom_s1(N, H, W, Ci, 3)
        ks0 = ops.choose_ksplit(g, Co)
        print(f"-- {Ci}->{Co} @ {H}x{W}: choose_ksplit = {ks0}")
        for ks in sorted({max(1, ks0 // 2), ks0, ks0 * 2, 4, 16}):
            bench_wgrad(N, H, W, Ci, Co, 3, ks)
    return True


def group_tinybench():
    """first / last layers (3 -> 128 fat-pixel conv, 128 -> 3 NCHW fp32 conv) at 256^2, N=32: fwd and fwd+bwd time"""
    import ops
    torch.manual_seed(0)
    N, H = 32, 256
    x = (torch.rand(N, 3, H, H, device=dev) - 0.5)
    wt = ((torch.rand(128, 3, 3, 3, device=dev) - 0.5) * 0.5).requires_grad_(True)
    b = rnd(128).requires_grad_(True)
    cache = ops.PackedCache()
    xa = ops.to_nhwc(x, None, None, True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timeit(fn, tag, iters=10):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        print(f"BENCH {tag}: {e0.elapsed_time(e1) / iters:.3f} ms", flush=True)

    with torch.no_grad():
        timeit(lambda: ops.conv(xa, wt, b, cache, "fat3"), "conv_in 3->128 fat3 fwd")
    gy = rnd(N, H, H, 128).to(torch.bfloat16)

    def fb():
        y = ops.conv(xa, wt, b, cache, "fat3")
        y.backward(gy)
    timeit(fb, "conv_in 3->128 fat3 fwd+bwd (wgrad only)")
    h = rnd(N, H, H, 128).to(torch.bfloat16).requires_grad_(True)
    w2 = (rnd(3, 128, 3, 3) * 0.03).requires_grad_(True)
    b2 = rnd(3).requires_grad_(True)
    c2 = ops.PackedCache()
    with torch.no_grad():
        timeit(lambda: ops.conv(h, w2, b2, c2, "s1", nchw_out=True), "conv_out 128->3 nchw fwd")
    g2 = rnd(N, 3, H, H)

    def fb2():
        y = ops.conv(h, w2, b2, c2, "s1", nchw_out=True)
        y.backward(g2)
    timeit(fb2, "conv_out 128->3 fwd+bwd (dgrad + wgrad)")
    return True


def group_bench():
    bench_conv(8, 64, 64, 512, 512, 3)
    bench_conv(8, 256, 256, 128, 128, 3)
    bench_conv(8, 128, 128, 256, 256, 3)
    bench_conv(8, 32, 32, 512, 512, 3)
    bench_conv(8, 128, 128, 512, 256, 1)
    bench_wgrad(8, 64, 64, 512, 512, 3, 4)
    bench_wgrad(8, 256, 256, 128, 128, 3, 32)
    bench_wgrad(8, 128, 128, 256, 256, 3, 8)
    return True


if __name__ == "__main__":
    grp = sys.argv[1]
    t0 = time.time()
    print(f"== group {grp}: device_ok={L.vqb_device_ok()} {torch.cuda.get_device_name(0)}", flush=True)
    ok = globals()["group_" + grp]()
    print(f"== group {grp} {'ALL PASS' if ok else 'HAS FAILURES'} in {time.time() - t0:.1f}s launches={native.launch_count()}",
          flush=True)
    sys.exit(0 if ok else 1)
