"""GPU (-m gpu): element-wise bounds of the video autoencoder's gradient GEMMs against float64, in the style and with the
helpers of test_gpu_kernel_bounds.py: |got - y64| <= u_out |y64| + tau S (tau = 2^-16, S = the same op on absolute
values), outputs in NaN-sentinel buffers with 4 KB guard bands (every addressed element written, nothing else touched),
inputs surrounded by NaN and with NaN channels past C inside a wider channel stride.

  vqb_conv3d_dgrad_gemm  the 64-tap data gradient of the folded up-sampling over the 8 parity views of dy
  vqb_conv3d_gemm        the Downsample data gradient: 8 parity-class launches writing strided sub-grids of one dx
  vqb_wgrad3d_gemm       s1, s2 and the 8-phase up-sampling weight gradient (ld_override / col_offset), its partial
                         buffer and the OIDHW split reduction (vqb_wgrad_reduce / vqb_wgrad_reduce_fold)
"""
import pytest
import torch

from test_gpu_kernel_bounds import (DEV, GUARD_BYTES, TAU, U_BF16, U_F32, Guarded, K, check, check_bits,  # noqa: F401
                                    check_stores, gather, gemm_truth, lib, ok, poisoned, rejects, rnd, stream,
                                    strided_index, views3d)

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- data gradients
@pytest.mark.parametrize("shp,Cy,Cx", [((1, 1, 1, 1), 8, 8), ((2, 2, 5, 3), 72, 136), ((1, 3, 2, 9), 136, 3),
                                       ((1, 2, 1, 130), 256, 72)])
def test_up_dgrad_64_taps_bounds(shp, Cy, Cx):
    """dx [N, t, h, w] from dy [N, 2t, 2h, 2w] (channel stride Cy + 8, NaN past Cy) through the 64-tap descriptor."""
    P, L = K.plans, K.L
    gen = torch.Generator(device=DEV).manual_seed(sum(shp) + Cy + Cx)
    N, t, h, w = shp
    Cys = Cy + 8
    DY = poisoned(rnd(N, 2 * t, 2 * h, 2 * w, Cy, gen=gen), Cys)
    g = P.geom3_up_dgrad(N, t, h, w, Cys)
    g.C = Cy
    assert len(g.taps) == 64
    Wg = poisoned(rnd(Cx, 64 * Cy, scale=(64 * Cy) ** -0.5, gen=gen), 64 * Cy)
    Cxs = P.cpad(Cx)
    strides = P.nthwc_strides(t, h, w, Cxs)
    d = P.conv3d_dgrad_desc(g, Cx, strides)
    total = N * t * h * w * Cxs

    def launch(wg=Wg):
        out = Guarded(total, torch.bfloat16)
        ok(L.vqb_conv3d_dgrad_gemm(d, DY.ptr(), wg.ptr(), out.ptr(), stream()), "conv3d_dgrad_gemm")
        torch.cuda.synchronize()
        return out

    out = launch()
    name = f"up dgrad 64 taps {shp} Cy={Cy} Cx={Cx}"
    idx = strided_index(0, (N, t, h, w, Cx), strides)
    check_stores(out, idx, name + " stores")
    vw, tp = views3d(g)
    wp = Wg.body.double().view(Cx, -1)
    y, S = gemm_truth(DY.body.double(), vw, tp, Cy, (N, t, h, w), wp)
    bound = U_BF16 * y.abs() + TAU["conv3d"] * S
    check(name, out.body[idx], y, bound, acc=(U_BF16 * y.abs(), TAU["conv3d"] * S))
    check_bits(name, out.bits(), launch().bits())
    if shp == (2, 2, 5, 3):  # the bound bites: one tap of one dx channel zeroed in the packed weights
        wm = Guarded(Wg.n, torch.bfloat16, poison="nan")
        wm.body.copy_(Wg.body)
        wm.body.view(Cx, -1)[Cx - 1, 63 * Cy:64 * Cy] = 0
        rejects("up dgrad: last tap of the last dx channel zeroed", launch(wm).body[idx], y, bound)


@pytest.mark.parametrize("shp,Cy,Cx", [((1, 2, 2, 2), 8, 8), ((2, 4, 10, 6), 136, 72), ((1, 6, 2, 130), 72, 3)])
def test_s2_dgrad_parity_classes_bounds(shp, Cy, Cx):
    """The Downsample data gradient: one vqb_conv3d_gemm per parity class of dx, each writing its strided sub-grid."""
    P, L = K.plans, K.L
    gen = torch.Generator(device=DEV).manual_seed(sum(shp) * 7 + Cy)
    N, T, H, W = shp
    Cys = Cy + 8
    DY = poisoned(rnd(N, T // 2, H // 2, W // 2, Cy, gen=gen), Cys)
    Cxs = P.cpad(Cx)
    total = N * T * H * W * Cxs
    classes = P.geom3_s2_dgrad_classes(N, T, H, W, Cys)
    runs = []
    for pt, ph, pw, g in classes:
        g.C = Cy
        n = len(g.taps)
        wg = poisoned(rnd(Cx, n * Cy, scale=(n * Cy) ** -0.5, gen=gen), n * Cy)
        strides, off = P.s2_dgrad_out(T, H, W, Cxs, pt, ph, pw)
        runs.append((g, wg, P.conv3d_desc(g, Cx, strides), off, strides))

    def launch():
        out = Guarded(total, torch.bfloat16)
        for g, wg, d, off, _ in runs:
            ok(L.vqb_conv3d_gemm(d, DY.ptr(), wg.ptr(), 0, 0, out.ptr(off), stream()), "conv3d_gemm s2 dgrad")
        torch.cuda.synchronize()
        return out

    out = launch()
    name = f"s2 dgrad classes {shp} Cy={Cy} Cx={Cx}"
    grid = (N, T // 2, H // 2, W // 2)
    idxs = [strided_index(off, grid + (Cx,), strides) for _, _, _, off, strides in runs]
    check_stores(out, torch.cat([i.reshape(-1) for i in idxs]), name + " stores")
    flat = DY.body.double()
    for (g, wg, _, _, _), idx, (pt, ph, pw, _) in zip(runs, idxs, classes):
        vw, tp = views3d(g)
        y, S = gemm_truth(flat, vw, tp, Cy, grid, wg.body.double().view(Cx, -1))
        check(f"{name} class {(pt, ph, pw)}", out.body[idx], y, U_BF16 * y.abs() + TAU["conv3d"] * S,
              acc=(U_BF16 * y.abs(), TAU["conv3d"] * S))
    check_bits(name, out.bits(), launch().bits())


# ---------------------------------------------------------------------------------------------------- weight gradient
WGRAD3_CASES = [
    # kind, (N, T, H, W) of x, C, Cout, ksplit
    ("s1", (1, 1, 1, 1), 8, 8, 3),
    ("s1", (2, 3, 5, 3), 72, 72, 1),
    ("s1", (1, 2, 1, 130), 136, 136, 3),
    ("s2", (1, 2, 2, 2), 72, 136, 5),
    ("s2", (2, 4, 10, 6), 8, 256, 1),
    ("up", (1, 1, 1, 1), 136, 72, 4),
    ("up", (2, 2, 5, 3), 8, 136, 1),
    ("up", (1, 3, 2, 9), 72, 256, 3),
]


@pytest.mark.parametrize("kind,shp,C,Cout,ksplit", WGRAD3_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_wgrad3d_bounds(kind, shp, C, Cout, ksplit):
    P, L = K.plans, K.L
    gen = torch.Generator(device=DEV).manual_seed(sum(shp) + C + Cout)
    N, T, H, W = shp
    Cs, Cys = C + 8, Cout + 8
    X = poisoned(rnd(N, T, H, W, C, gen=gen), Cs)
    C64 = (C + 63) // 64 * 64
    if kind == "up":
        phases = [(a, b, e) for a in range(2) for b in range(2) for e in range(2)]
        geoms = [P.geom3_up_fwd(N, T, H, W, Cs, *ph) for ph in phases]
        dyshape = (N, 2 * T, 2 * H, 2 * W)
    else:
        geoms = [(P.geom3_s2 if kind == "s2" else P.geom3_s1)(N, T, H, W, Cs)]
        dyshape = (N, geoms[0].To, geoms[0].Ho, geoms[0].Wo)
    for g in geoms:
        g.C = C
    DY = poisoned(rnd(*dyshape, Cout, gen=gen), Cys)
    ntaps = len(geoms[0].taps)
    cols = L.vqb_wgrad_cols(ntaps, C)
    if kind == "up":
        ld = 64 * C64
        descs = [P.wgrad3d_desc(g, Cout, ksplit, dy_view=P.up3_dy_view(N, T, H, W, Cys, *ph), ld_override=ld,
                                col_offset=p * 8 * C64) for p, (g, ph) in enumerate(zip(geoms, phases))]
    else:
        ld = cols
        descs = [P.wgrad3d_desc(geoms[0], Cout, ksplit, dy_view=K.native.dense_view3d(*dyshape, Cys))]

    def launch():
        part = Guarded(ksplit * Cout * ld, torch.float32)
        for d in descs:
            ok(L.vqb_wgrad3d_gemm(d, DY.ptr(), X.ptr(), part.ptr(), stream()), f"wgrad3d_gemm {kind}")
        torch.cuda.synchronize()
        return part

    part = launch()
    name = f"wgrad3d {kind} {shp} C={C} Cout={Cout} ksplit={ksplit}"
    written = torch.cat([strided_index(d.col_offset, (ksplit, Cout, cols), (Cout * ld, ld, 1)).reshape(-1)
                         for d in descs])
    check_stores(part, written, name + " partial stores")
    xf, dyf = X.body.double(), DY.body.double()
    ref = torch.zeros(Cout, len(geoms) * ntaps, C, device=DEV, dtype=torch.float64)
    S = torch.zeros_like(ref)
    for p, (g, d) in enumerate(zip(geoms, descs)):
        dv = d.dy_view
        grid = (g.N, g.To, g.Ho, g.Wo)
        dy = gather(dyf, dv.offset, (dv.Nv, dv.Tv, dv.Hv, dv.Wv), (dv.sn, dv.st, dv.sh, dv.sw), Cout, grid, (0, 0, 0, 0))
        vw, tp = views3d(g)
        for tt, (v, shift) in enumerate(tp):
            a = gather(xf, *vw[v], C, grid, shift)
            ref[:, p * ntaps + tt] = dy.reshape(-1, Cout).t() @ a.reshape(-1, C)
            S[:, p * ntaps + tt] = dy.abs().reshape(-1, Cout).t() @ a.abs().reshape(-1, C)
    pv = part.body.view(ksplit, Cout, ld)[:, :, :len(geoms) * cols].reshape(ksplit, Cout, -1, C64)
    tau = TAU["wgrad"]
    bound = U_F32 * ref.abs() + tau * S
    check(name + " partial", pv.double().sum(0)[:, :, :C], ref, bound, acc=(U_F32 * ref.abs(), tau * S))
    if C64 > C:  # the C64 padding columns read TMA zero fill only
        check(name + " partial C64 padding columns", pv[:, :, :, C:], torch.zeros_like(pv[:, :, :, C:]), 0.0)
    check_bits(name + " partial", part.bits(), launch().bits())
    if kind == "s1" and shp == (2, 3, 5, 3):  # the bound bites
        g_m = pv.double().sum(0)[:, :, :C].clone()
        g_m[Cout - 1, 13] = 0
        rejects("wgrad3d: centre tap of the last output channel zeroed", g_m, ref, bound)
    # split reduction to OIDHW (27 taps; the up-sampling's 64 folded slots through the tap masks)
    if kind == "up":
        masks = [m for g in geoms for m in g.tapmask]
        tm = torch.tensor(masks, device=DEV, dtype=torch.int32)
        sel = torch.tensor([[(m >> q) & 1 for q in range(27)] for m in masks], device=DEV, dtype=torch.float64)
    else:
        tm = torch.tensor(geoms[0].tapmap, device=DEV, dtype=torch.int32)
        sel = torch.nn.functional.one_hot(tm.long(), 27).double()
    gref = torch.einsum("osc,st->oct", ref, sel)
    gS = torch.einsum("osc,st->oct", S, sel)
    grad = Guarded(Cout * C * 27, torch.float32)
    nslots = len(geoms) * ntaps
    if kind == "up":
        ok(L.vqb_wgrad_reduce_fold(part.ptr(), grad.ptr(), ksplit, Cout, Cout, C, 27, nslots, C64, tm.data_ptr(),
                                   stream()), "wgrad_reduce_fold")
    else:
        ok(L.vqb_wgrad_reduce(part.ptr(), grad.ptr(), ksplit, Cout, Cout, C, 27, nslots, C64, tm.data_ptr(), 0,
                              stream()), "wgrad_reduce")
    torch.cuda.synchronize()
    check_stores(grad, torch.arange(grad.n, device=DEV), name + " reduce stores")
    psum = pv.double().abs().sum(0)[:, :, :C]
    b = U_F32 * gref.abs() + tau * gS + ksplit * U_F32 * torch.einsum("osc,st->oct", psum, sel)
    check(name + " reduce", grad.body.view(Cout, C, 27), gref, b)
