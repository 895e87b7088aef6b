"""GPU (-m gpu): element-wise bounds of every native kernel against a float64 reference of the same operation.

Each case runs one C ABI entry point on bf16 inputs and compares every output element with the same operation in float64
on exactly the values the kernel read (the bf16 inputs and the packed bf16 weights are exact in float64):

  GEMM-like outputs (conv, dgrad, conv3d, wgrad)  |got - y64| <= u_out |y64| + tau S,  S = the same op on |x|, |w| (+ |bias|
                                                   + |res|): the standard bound on the accumulation error; u_out = 2^-8
                                                   for bf16 outputs, 2^-24 for fp32 outputs
  attention                                        |o - o64| <= 2^-8 |o64| + 2^-8 SDPA64(q, k, |v|)  (P is rounded to bf16
                                                   before P.V); lse against the fp64 log-sum-exp; dq, dk, dv per
                                                   (n, head, token) row within 2^-6 of the row's fp64 norm
  GroupNorm (+ SiLU)                               one bf16 rounding + the MUFU.TANH sigmoid + a statistics term; mean /
                                                   rstd, dgamma, dbeta and dx_colsum against fp64
  layout, pack, max-pool                           bit-exact where the header promises an exact copy

Outputs are views into a larger buffer pre-filled with a NaN sentinel bit pattern (4 KB guard bands on both sides):
every element the descriptor addresses must be overwritten and every other element (guard bands, pad channels, other
parity phases, frames) must still hold the exact sentinel bits. Inputs are surrounded by NaN, and channels past a view's
C inside a wider-stride tensor are NaN, so an over-read shows up as a NaN in the output. The fat-pixel first layer is
the exception its contract states: it reads the zero frame and the 64 zeroed slack elements (plans.FAT_K), so only
memory beyond those is poisoned.

Mutation checks prove that the bounds bite: the same checker must reject a kernel output with one packed tap of one
output channel zeroed, a reference computed without the last 8 channels of the last K-chunk, a last-tile output with one
tap's contribution removed at one voxel, an attention reference with two keys of the ragged tail swapped, and GroupNorm
references with a wrong statistic. Kernels documented as deterministic (no atomics) are run twice and must agree bit for
bit.

`python -m pytest -m gpu -q tests/test_gpu_kernel_bounds.py -s` prints one line per case with max(err/bound).
"""
import math
import types

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# Accumulation-error factor tau of the GEMM bound, per kernel family, set at 2^-16 before any measurement. Next to each
# value: the largest "accumulation share" max((err - u_out |y64|)+ / (tau S)) this file observed on one H100 80GB HBM3
# (700 W power limit). All are well below 1, so tau stays at 2^-16 (observed accumulation error <= 2^-21 S).
TAU = {
    "conv": 2.0 ** -16,  # 0.027
    "conv3d": 2.0 ** -16,  # 0.033
    "wgrad": 2.0 ** -16,  # 0.017
}

U_BF16 = 2.0 ** -8
U_F32 = 2.0 ** -24
GUARD_BYTES = 4096
SENTINEL = {torch.bfloat16: 0x7F81, torch.float32: 0x7FC0DEAD}  # NaN payloads no kernel produces
BITS = {torch.bfloat16: torch.int16, torch.float32: torch.int32}
DEV = "cuda"

K = types.SimpleNamespace(L=None, native=None, plans=None)


@pytest.fixture(scope="module", autouse=True)
def lib():
    """Loads the native library lazily so that a machine without a GPU collects this file and skips it cleanly."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import native
    import plans

    L = native.load()
    if not L.vqb_device_ok():
        pytest.skip("needs an sm_90 device")
    K.L, K.native, K.plans = L, native, plans
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield L
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def stream():
    return torch.cuda.current_stream().cuda_stream


def ok(rc, what):
    K.native.check(rc, what)


# ---------------------------------------------------------------------------------------------------- guarded memory
class Guarded:
    """A flat device buffer [guard | body | guard]; the guards hold the sentinel (outputs) or NaN (inputs)."""

    def __init__(self, numel, dtype, poison="sentinel"):
        self.dtype = dtype
        self.es = torch.tensor([], dtype=dtype).element_size()
        self.g = GUARD_BYTES // self.es
        self.n = int(numel)
        self.buf = torch.empty(self.n + 2 * self.g, device=DEV, dtype=dtype)
        if poison == "sentinel":
            self.buf.view(BITS[dtype]).fill_(SENTINEL[dtype])
        else:
            self.buf.fill_(float("nan"))

    @property
    def body(self):
        return self.buf[self.g:self.g + self.n]

    def ptr(self, off=0):
        return self.buf.data_ptr() + (self.g + int(off)) * self.es

    def bits(self):
        return self.buf.view(BITS[self.dtype]).clone()


def strided_index(offset, shape, strides):
    idx = torch.full((), int(offset), dtype=torch.long, device=DEV)
    for e, s in zip(shape, strides):
        idx = idx.unsqueeze(-1) + torch.arange(int(e), device=DEV, dtype=torch.long) * int(s)
    return idx


def check_stores(G, written, what):
    """Every element of `written` (body indices) was overwritten; every other element still holds the sentinel."""
    sent = G.buf.view(BITS[G.dtype]) == SENTINEL[G.dtype]
    mask = torch.zeros_like(sent)
    mask[G.g + written.reshape(-1)] = True
    missed = (mask & sent).nonzero()
    assert missed.numel() == 0, f"{what}: {missed.numel()} addressed elements were not written (first at body index " \
                                f"{missed[0].item() - G.g})"
    stray = (~mask & ~sent).nonzero()
    assert stray.numel() == 0, f"{what}: {stray.numel()} elements outside the addressed set were written (first at " \
                               f"body index {stray[0].item() - G.g} of {G.n})"


def poisoned(vals, Cs):
    """vals [..., C] -> NaN-guarded buffer with channel stride Cs >= C; channels C..Cs-1 are NaN."""
    *lead, C = vals.shape
    G = Guarded(math.prod(lead) * Cs, vals.dtype, poison="nan")
    G.body.view(*lead, Cs)[..., :C] = vals
    return G


def rnd(*shape, scale=1.0, dtype=torch.bfloat16, gen=None):
    return (torch.randn(*shape, device=DEV, generator=gen) * scale).to(dtype)


# ---------------------------------------------------------------------------------------------------- the checker
def worst(got, truth, bound):
    """-> (max err/bound, description of the worst element). A zero bound admits only an exact match."""
    got = got.double()
    truth = truth.double()
    bound = torch.as_tensor(bound, device=DEV, dtype=torch.float64).expand_as(truth)
    bad = ~torch.isfinite(got)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        return math.inf, f"non-finite output at {i}: got={got[tuple(i)].item()} truth={truth[tuple(i)].item()}"
    err = (got - truth).abs()
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    j = int(ratio.reshape(-1).argmax())
    i = [int(v) for v in torch.unravel_index(torch.tensor(j), ratio.shape)]
    r = ratio.reshape(-1)[j].item()
    return r, (f"worst element {i}: got={got.reshape(-1)[j].item():.7g} truth={truth.reshape(-1)[j].item():.7g} "
               f"bound={bound.reshape(-1)[j].item():.3g}")


def check(name, got, truth, bound, acc=None):
    """acc = (u_out |y64|, tau S): also print max((err - u_out |y64|)+ / (tau S)), the share of the accumulation term."""
    r, info = worst(got, truth, bound)
    if acc is not None and math.isfinite(r):
        rnd_part, acc_part = acc
        e = ((got.double() - truth).abs() - rnd_part).clamp_min(0)
        info += f"  accumulation share={(e / acc_part.clamp_min(1e-300)).max().item():.3g}"
    print(f"  {name}: max(err/bound)={r:.3g}  {info}", flush=True)
    assert r <= 1.0, f"{name}: max(err/bound)={r:.3g}, {info}"
    return r


def rejects(name, got, truth, bound):
    r, info = worst(got, truth, bound)
    print(f"  mutation {name}: rejected={r > 1.0} (max(err/bound)={r:.3g})", flush=True)
    assert r > 1.0, f"mutation {name} was accepted by the checker (max(err/bound)={r:.3g}): the bound is too loose"


def check_bits(name, a, b):
    same = torch.equal(a, b)
    print(f"  {name}: run-twice bit-identical={same}", flush=True)
    assert same, f"{name}: two runs of a deterministic kernel differ"


def bf16_ulp(x):
    """One bf16 ulp at |x| (the spacing of bf16 values around x), >= the smallest normal's."""
    m, e = torch.frexp(x.double().abs())
    return torch.ldexp(torch.ones_like(m), (e - 8).clamp_min(-133))


# ---------------------------------------------------------------------------------------------------- GEMM reference
def gather(flat, off, vext, vstr, C, grid, shift):
    """Tap operand: A_view[n, t + dt, h + dh, w + dw, :C] over the output grid, zero out of range (TMA zero fill)."""
    Av = flat.as_strided(tuple(vext) + (C,), tuple(vstr) + (1,), int(off))
    out = flat.new_zeros(tuple(grid) + (C,))
    so, si = [], []
    for e, gsz, s in zip(vext, grid, shift):
        lo, hi = max(0, -s), min(gsz, e - s)
        if hi <= lo:
            return out
        so.append(slice(lo, hi))
        si.append(slice(lo + s, hi + s))
    out[tuple(so)] = Av[tuple(si)]
    return out


def views2d(g):
    return [(v.offset, (v.Nv, v.Hv, v.Wv), (v.sn, v.sh, v.sw)) for v in g.views], \
           [(t[0], (0, t[2], t[1])) for t in g.taps]


def views3d(g):
    return [(v.offset, (v.Nv, v.Tv, v.Hv, v.Wv), (v.sn, v.st, v.sh, v.sw)) for v in g.views], \
           [(t[0], (0, t[3], t[2], t[1])) for t in g.taps]


def gemm_truth(flat, views, taps, C, grid, wp):
    """y64[..., co] = sum_t sum_c A_t[..., c] wp[co, t*C + c] and the same on absolute values."""
    Cout = wp.shape[0]
    y = flat.new_zeros(tuple(grid) + (Cout,))
    S = torch.zeros_like(y)
    for t, (v, shift) in enumerate(taps):
        a = gather(flat, *views[v], C, grid, shift)
        w = wp[:, t * C:(t + 1) * C]
        y += a @ w.t()
        S += a.abs() @ w.abs().t()
    return y, S


# ---------------------------------------------------------------------------------------------------- 2-D conv
BN_COUTS = {16: (3, 8, 16), 32: (24, 32), 64: (40, 64), 128: (72, 128, 136, 320)}
CS2D = (8, 24, 64, 72, 136, 512)
SHAPES2D = ((1, 1, 1), (3, 1, 130), (11, 4, 4), (2, 5, 3), (1, 256, 256), (8, 64, 64))
EPIS = ("bias", "res", "relu+bias", "mask", "bias+res+relu", "", "res+mask")
STORES = ("nhwc", "nchw32", "nhwc", "nchw16")


def conv2d_cases():
    cases = []
    k = 0
    for i, shp in enumerate(SHAPES2D):
        for j, bn in enumerate(BN_COUTS):
            cout = BN_COUTS[bn][(i + j) % len(BN_COUTS[bn])]
            cs = CS2D if shp[0] * shp[1] * shp[2] < 32768 else CS2D[:5]
            C = cs[(i + 2 * j) % len(cs)]
            cases.append(("s1", shp, C, cout, EPIS[k % len(EPIS)], STORES[k % 4]))
            k += 1
    for i, shp in enumerate(SHAPES2D):  # 1x1
        bn = list(BN_COUTS)[i % 4]
        cases.append(("p1", shp, CS2D[(i + 3) % 6] if i < 4 else 64, BN_COUTS[bn][-1], EPIS[i % len(EPIS)],
                      STORES[(i + 1) % 4]))
    for j, bn in enumerate(BN_COUTS):  # stride 2 over 2x2 inputs, and larger
        cases.append(("s2", (1, 2, 2), CS2D[j], BN_COUTS[bn][0], "bias", "nhwc"))
        cases.append(("s2", ((11, 8, 8), (3, 2, 260), (2, 10, 6), (2, 64, 64))[j], (72, 136, 24, 64)[j],
                      BN_COUTS[bn][-1], EPIS[j], STORES[j]))
    for j, bn in enumerate(BN_COUTS):  # stride-1 data gradient
        cases.append(("dg1", SHAPES2D[(j + 1) % 6], (72, 64, 136, 24)[j], BN_COUTS[bn][0], "mask" if j % 2 else "",
                      "nhwc"))
    for j, bn in enumerate(BN_COUTS):  # stride-2 data gradient: one parity class per launch
        cases.append((f"dg2{j >> 1}{j & 1}", ((11, 8, 8), (3, 2, 260), (2, 6, 6), (1, 2, 2))[j], (64, 72, 8, 136)[j],
                      BN_COUTS[bn][-1], "", "nhwc"))
    for j, bn in enumerate(BN_COUTS):  # folded nearest-2x up-sampling, one phase per launch
        cases.append((f"up{j >> 1}{j & 1}", ((11, 4, 4), (3, 1, 130), (2, 5, 3), (1, 1, 1))[j], (136, 64, 72, 24)[j],
                      BN_COUTS[bn][j % len(BN_COUTS[bn])], "bias", "nhwc"))
    for j, bn in enumerate(BN_COUTS):  # first-layer fat-pixel conv over the zero-framed 8-channel image
        cases.append(("fat3" if j < 3 else "fatdg", ((2, 5, 3), (3, 1, 130), (8, 64, 64), (1, 1, 1))[j], 64,
                      BN_COUTS[bn][0], ("bias", "", "bias", "mask")[j], "nhwc"))
    # GroupNorm statistics in the epilogue (whole tiles inside one image, Cout % 64 == 0)
    cases.append(("s1", (2, 16, 16), 64, 64, "stats+bias", "nhwc"))
    cases.append(("s1", (8, 64, 64), 72, 320, "stats+res", "nhwc"))
    cases.append(("up11", (2, 16, 16), 64, 128, "stats+bias", "nhwc"))
    return cases


def build_conv2d(kind, shp, C, Cout, epi, store, seed=0):
    P = K.plans
    gen = torch.Generator(device=DEV).manual_seed(seed)
    N, H, W = shp
    Cs = C + 8  # a wider-stride tensor: channels C..Cs-1 must never be read
    fat = kind in ("fat3", "fatdg")
    if fat:
        n = N * (H + 2) * (W + 2) * 8
        A = Guarded(n + P.FAT_K, torch.bfloat16, poison="nan")
        A.body.zero_()  # zero frame + zeroed slack are part of the contract
        A.body[:n].view(N, H + 2, W + 2, 8)[:, 1:-1, 1:-1, :] = rnd(N, H, W, 8, gen=gen)
        g = P.geom_fat3(N, H, W, dgrad=kind == "fatdg")
        Ccol = P.FAT_K
    else:
        if kind in ("s1", "p1", "dg1"):
            lead = (N, H, W)
            g = P.geom_s1_dgrad(N, H, W, Cs, 3) if kind == "dg1" else P.geom_s1(N, H, W, Cs, 1 if kind == "p1" else 3)
        elif kind == "s2":
            lead = (N, H, W)
            g = P.geom_s2(N, H, W, Cs)
        elif kind.startswith("dg2"):
            lead = (N, H // 2, W // 2)
            ph, pw = int(kind[3]), int(kind[4])
            g = P.geom_s2_dgrad_classes(N, H, W, Cs)[ph * 2 + pw][2]
        else:  # up phase over the low-resolution input
            lead = (N, H, W)
            ph, pw = int(kind[2]), int(kind[3])
            g = P.geom_up_fwd(N, H, W, Cs, ph, pw)
        A = poisoned(rnd(*lead, C, gen=gen), Cs)
        g.C = C
        Ccol = C
    ntaps = len(g.taps)
    wv = rnd(Cout, ntaps, Ccol, scale=(ntaps * Ccol) ** -0.5, gen=gen)
    if fat:
        wv[:, :, 24:] = 0  # columns 24..63 of a fat tap meet the next pixels and carry zero weights
    Wg = poisoned(wv.reshape(Cout, ntaps * Ccol), ntaps * Ccol)
    Cso = P.cpad(Cout)
    grid = (g.N, g.Ho, g.Wo)
    off = 0
    if store == "nhwc":
        if kind.startswith("dg2"):
            total = N * H * W * Cso
            strides = (H * W * Cso, 2 * W * Cso, 2 * Cso, 1)
            off = (ph * W + pw) * Cso
        elif kind.startswith("up"):
            total = N * 4 * H * W * Cso
            strides = (4 * H * W * Cso, 4 * W * Cso, 2 * Cso, 1)
            off = (ph * 2 * W + pw) * Cso
        else:
            total = g.N * g.Ho * g.Wo * Cso
            strides = P.nhwc_strides(g.Ho, g.Wo, Cso)
    else:
        total = g.N * Cout * g.Ho * g.Wo
        strides = P.nchw_strides(Cout, g.Ho, g.Wo)
    out_f32 = store == "nchw32"
    odt = torch.float32 if out_f32 else torch.bfloat16
    idx = strided_index(off, grid + (Cout,), strides)
    flags = 0
    bias = res = mask = stats = None
    if "bias" in epi:
        flags |= K.native.EPI_BIAS
        bias = Guarded(Cout, torch.float32, poison="nan")
        bias.body.copy_(torch.randn(Cout, device=DEV, generator=gen))
    if "res" in epi:
        flags |= K.native.EPI_RES
        res = Guarded(total, torch.bfloat16, poison="nan")
        res.body[idx] = rnd(*idx.shape, gen=gen)
    if "mask" in epi:
        flags |= K.native.EPI_MASK
        mask = Guarded(total, torch.bfloat16, poison="nan")
        mask.body[idx] = rnd(*idx.shape, gen=gen)
    if "relu" in epi:
        flags |= K.native.EPI_RELU
    if "stats" in epi:
        flags |= K.native.EPI_STATS
    d = P.conv_desc(g, Cout, strides, flags, out_f32)
    d.C = Ccol
    if "stats" in epi:
        assert K.L.vqb_conv_stats_ok(d) == 1, "statistics case is not a supported shape"

    def launch(wg=Wg):
        out = Guarded(total, odt)
        st = None
        if "stats" in epi:
            st = Guarded(g.N * Cout * 2, torch.float32)
            st.body.zero_()
        ok(K.L.vqb_conv_gemm(d, A.ptr(), wg.ptr(), bias.ptr() if bias else 0, res.ptr(off) if res else 0,
                             mask.ptr(off) if mask else 0, out.ptr(off), st.ptr() if st else 0, stream()),
           f"conv_gemm {kind}")
        torch.cuda.synchronize()
        return out, st

    vw, tp = views2d(g)
    flat = A.body.double()

    def truth(wp64):
        y, S = gemm_truth(flat, vw, tp, Ccol, grid, wp64)
        if bias is not None:
            y = y + bias.body.double()
            S = S + bias.body.double().abs()
        if res is not None:
            r = res.body[idx].double()
            y, S = y + r, S + r.abs()
        if "relu" in epi:
            y = y.clamp_min(0)
        if mask is not None:
            y = y * (mask.body[idx].double() > 0)
        return y, S

    return types.SimpleNamespace(g=g, A=A, Wg=Wg, wv=wv, launch=launch, truth=truth, idx=idx, grid=grid, vw=vw, tp=tp,
                                 flat=flat, Ccol=Ccol, Cout=Cout, u=U_F32 if out_f32 else U_BF16, total=total,
                                 odt=odt, stats="stats" in epi, N=g.N)


def conv_bound(c, y, S, tau):
    return c.u * y.abs() + tau * S


@pytest.mark.parametrize("kind,shp,C,Cout,epi,store", conv2d_cases(),
                         ids=lambda v: str(v).replace(" ", "") if not isinstance(v, str) else (v or "plain"))
def test_conv_gemm_bounds(kind, shp, C, Cout, epi, store):
    c = build_conv2d(kind, shp, C, Cout, epi, store)
    out, st = c.launch()
    name = f"conv {kind} {shp} C={C} Cout={Cout} {epi or 'plain'} {store}"
    check_stores(out, c.idx, name + " stores")
    got = out.body[c.idx]
    y, S = c.truth(c.Wg.body.double().view(c.Cout, -1))
    check(name, got, y, conv_bound(c, y, S, TAU["conv"]), acc=(c.u * y.abs(), TAU["conv"] * S))
    if c.stats:
        check_stores(st, torch.arange(st.n, device=DEV), name + " stats stores")
        v = got.double()
        red = tuple(range(1, v.dim() - 1))
        ref = torch.stack([v.sum(red), (v * v).sum(red)], -1)  # [N, Cout, 2] of the bf16 values written
        absr = torch.stack([v.abs().sum(red), (v * v).sum(red)], -1)
        depth = 64 + math.prod(c.grid[1:]) // 128  # fp32 adds in the longest chain: warp + tile tree + atomics
        check(name + " EPI_STATS sums", st.body.view(c.N, c.Cout, 2), ref, depth * U_F32 * absr)
    else:
        out2, _ = c.launch()
        check_bits(name, out.bits(), out2.bits())


def test_conv_mutations_rejected():
    """The conv checker rejects: one zeroed packed tap of one output channel; a reference without the last 8 channels of
    the last K-chunk; the last ragged tile with one tap's contribution removed at one voxel."""
    c = build_conv2d("s1", (3, 1, 130), 72, 136, "bias", "nhwc", seed=5)
    out, _ = c.launch()
    wp = c.Wg.body.double().view(c.Cout, -1)
    y, S = c.truth(wp)
    got = out.body[c.idx]
    check("conv s1 (3,1,130) C=72 Cout=136 (mutation base)", got, y, conv_bound(c, y, S, TAU["conv"]))
    co, t = c.Cout - 1, 4
    wm = Guarded(c.Wg.n, torch.bfloat16, poison="nan")
    wm.body.copy_(c.Wg.body)
    wm.body.view(c.Cout, -1)[co, t * c.Ccol:(t + 1) * c.Ccol] = 0
    out_m, _ = c.launch(wm)
    rejects("conv: packed tap 4 of the last output channel zeroed", out_m.body[c.idx], y, conv_bound(c, y, S,
                                                                                                      TAU["conv"]))
    wcut = wp.clone().view(c.Cout, 9, c.Ccol)
    wcut[:, :, c.Ccol - 8:] = 0
    y_m, S_m = c.truth(wcut.view(c.Cout, -1))
    rejects("conv: reference without the last 8 channels of the last K-chunk", got, y_m,
            conv_bound(c, y_m, S_m, TAU["conv"]))
    # last voxel of the last (ragged) tile: remove the centre tap's contribution from every output channel there
    v, shift = c.tp[4]
    a = gather(c.flat, *c.vw[v], c.Ccol, c.grid, shift)[-1, -1, -1]
    contrib = a @ wp[:, 4 * c.Ccol:5 * c.Ccol].t()
    got_m = got.clone()
    got_m[-1, -1, -1] = (got[-1, -1, -1].double() - contrib).to(torch.bfloat16)
    rejects("conv: last ragged tile, one tap removed at one voxel", got_m, y, conv_bound(c, y, S, TAU["conv"]))


# ---------------------------------------------------------------------------------------------------- 3-D conv
SHAPES3D = ((1, 1, 9, 21), (2, 5, 9, 21), (1, 6, 4, 4), (3, 2, 2, 2), (1, 3, 1, 130))
COUT3D = {16: (3, 16), 32: (32,), 64: (64,), 128: (72, 256)}
CS3D = (8, 64, 72, 136)


def conv3d_cases():
    cases = []
    k = 0
    for i, shp in enumerate(SHAPES3D):
        for j, bn in enumerate(COUT3D):
            cases.append(("s1", shp, CS3D[(i + j) % 4], COUT3D[bn][(i + j) % len(COUT3D[bn])],
                          ("bias", "res", "bias+res", "")[k % 4], ("nthwc", "ncthw32", "nthwc", "ncthw16")[k % 4]))
            k += 1
    for j, shp in enumerate(((1, 6, 4, 4), (3, 2, 2, 2), (2, 10, 18, 42), (1, 2, 2, 260))):  # stride-2 inputs
        cases.append(("s2", shp, CS3D[(j + 1) % 4], (72, 16, 256, 32)[j], ("bias", "res", "bias+res", "")[j],
                      ("nthwc", "ncthw16", "ncthw32", "nthwc")[j]))
    for j, shp in enumerate(((1, 1, 9, 21), (3, 2, 2, 2), (1, 3, 1, 130), (2, 5, 9, 21))):  # all 8 up-sampling phases
        cases.append(("up", shp, CS3D[j], (64, 256, 3, 32)[j], ("bias", "", "bias", "bias")[j], "nthwc"))
    cases.append(("up101", (1, 3, 4, 5), 72, 16, "bias", "nthwc"))  # one phase alone: the other 7 stay untouched
    return cases


def build_conv3d(kind, shp, C, Cout, epi, store, seed=0):
    P = K.plans
    gen = torch.Generator(device=DEV).manual_seed(seed)
    N, T, H, W = shp
    Cs = C + 8
    A = poisoned(rnd(N, T, H, W, C, gen=gen), Cs)
    Cso = P.cpad(Cout)
    if kind == "s1":
        geoms = [(P.geom3_s1(N, T, H, W, Cs), 0)]
    elif kind == "s2":
        geoms = [(P.geom3_s2(N, T, H, W, Cs), 0)]
    else:
        phases = [(a, b, e) for a in range(2) for b in range(2) for e in range(2)] if kind == "up" else \
                 [(int(kind[2]), int(kind[3]), int(kind[4]))]
        geoms = [(P.geom3_up_fwd(N, T, H, W, Cs, *ph), ((ph[0] * 2 * H + ph[1]) * 2 * W + ph[2]) * Cso)
                 for ph in phases]
    g0 = geoms[0][0]
    for g, _ in geoms:
        g.C = C
    ntaps = len(g0.taps)
    if kind.startswith("up"):
        total = N * 8 * T * H * W * Cso
        strides = P.up3_out_strides(T, H, W, Cso)
    elif store == "nthwc":
        total = N * g0.To * g0.Ho * g0.Wo * Cso
        strides = P.nthwc_strides(g0.To, g0.Ho, g0.Wo, Cso)
    else:
        total = N * Cout * g0.To * g0.Ho * g0.Wo
        strides = P.ncthw_strides(Cout, g0.To, g0.Ho, g0.Wo)
    out_f32 = store == "ncthw32"
    odt = torch.float32 if out_f32 else torch.bfloat16
    grid = (g0.N, g0.To, g0.Ho, g0.Wo)
    idxs = [strided_index(off, grid + (Cout,), strides) for _, off in geoms]
    flags = 0
    bias = res = None
    if "bias" in epi:
        flags |= K.native.EPI_BIAS
        bias = Guarded(Cout, torch.float32, poison="nan")
        bias.body.copy_(torch.randn(Cout, device=DEV, generator=gen))
    if "res" in epi:
        flags |= K.native.EPI_RES
        res = Guarded(total, torch.bfloat16, poison="nan")
        for idx in idxs:
            res.body[idx] = rnd(*idx.shape, gen=gen)
    Ws = []
    for _ in geoms:
        wv = rnd(Cout, ntaps * C, scale=(ntaps * C) ** -0.5, gen=gen)
        Ws.append(poisoned(wv, ntaps * C))
    descs = [P.conv3d_desc(g, Cout, strides, flags, out_f32) for g, _ in geoms]

    def launch(ws=None):
        ws = ws or Ws
        out = Guarded(total, odt)
        for d, (_, off), wg in zip(descs, geoms, ws):
            ok(K.L.vqb_conv3d_gemm(d, A.ptr(), wg.ptr(), bias.ptr() if bias else 0, res.ptr(off) if res else 0,
                                   out.ptr(off), stream()), f"conv3d_gemm {kind}")
        torch.cuda.synchronize()
        return out

    flat = A.body.double()
    vts = [views3d(g) for g, _ in geoms]

    def truth(p, wp64):
        vw, tp = vts[p]
        y, S = gemm_truth(flat, vw, tp, C, grid, wp64)
        if bias is not None:
            y, S = y + bias.body.double(), S + bias.body.double().abs()
        if res is not None:
            r = res.body[idxs[p]].double()
            y, S = y + r, S + r.abs()
        return y, S

    return types.SimpleNamespace(launch=launch, truth=truth, idxs=idxs, Ws=Ws, C=C, Cout=Cout, grid=grid, vts=vts,
                                 flat=flat, u=U_F32 if out_f32 else U_BF16, total=total, ntaps=ntaps)


@pytest.mark.parametrize("kind,shp,C,Cout,epi,store", conv3d_cases(),
                         ids=lambda v: str(v).replace(" ", "") if not isinstance(v, str) else (v or "plain"))
def test_conv3d_gemm_bounds(kind, shp, C, Cout, epi, store):
    c = build_conv3d(kind, shp, C, Cout, epi, store)
    out = c.launch()
    name = f"conv3d {kind} {shp} C={C} Cout={Cout} {epi or 'plain'} {store}"
    check_stores(out, torch.cat([i.reshape(-1) for i in c.idxs]), name + " stores")
    for p, idx in enumerate(c.idxs):
        y, S = c.truth(p, c.Ws[p].body.double().view(c.Cout, -1))
        check(name + (f" phase {p}" if len(c.idxs) > 1 else ""), out.body[idx], y,
              c.u * y.abs() + TAU["conv3d"] * S, acc=(c.u * y.abs(), TAU["conv3d"] * S))
    check_bits(name, out.bits(), c.launch().bits())


def test_conv3d_1x1x1_via_conv_gemm():
    """The 1x1x1 convs of the video model run through vqb_conv_gemm on the [N][T*H][W][C] view."""
    for shp, C, Cout in (((2, 5, 9, 21), 136, 72), ((1, 3, 1, 130), 64, 16)):
        N, T, H, W = shp
        c = build_conv2d("p1", (N, T * H, W), C, Cout, "bias+res", "nhwc", seed=7)
        out, _ = c.launch()
        name = f"conv3d 1x1x1 {shp} C={C} Cout={Cout} via [N][T*H][W][C]"
        check_stores(out, c.idx, name + " stores")
        y, S = c.truth(c.Wg.body.double().view(c.Cout, -1))
        check(name, out.body[c.idx], y, conv_bound(c, y, S, TAU["conv"]))


def test_conv3d_mutations_rejected():
    c = build_conv3d("s1", (1, 3, 1, 130), 72, 72, "bias", "nthwc", seed=9)
    out = c.launch()
    idx = c.idxs[0]
    wp = c.Ws[0].body.double().view(c.Cout, -1)
    y, S = c.truth(0, wp)
    bound = c.u * y.abs() + TAU["conv3d"] * S
    got = out.body[idx]
    check("conv3d s1 (1,3,1,130) C=72 Cout=72 (mutation base)", got, y, bound)
    wm = Guarded(c.Ws[0].n, torch.bfloat16, poison="nan")
    wm.body.copy_(c.Ws[0].body)
    wm.body.view(c.Cout, -1)[c.Cout - 1, 13 * c.C:14 * c.C] = 0
    rejects("conv3d: packed centre tap of the last output channel zeroed", c.launch([wm]).body[idx], y, bound)
    wcut = wp.clone().view(c.Cout, c.ntaps, c.C)
    wcut[:, :, c.C - 8:] = 0
    y_m, S_m = c.truth(0, wcut.view(c.Cout, -1))
    rejects("conv3d: reference without the last 8 channels of the last K-chunk", got, y_m,
            c.u * y_m.abs() + TAU["conv3d"] * S_m)
    vw, tp = c.vts[0]
    v, shift = tp[13]
    a = gather(c.flat, *vw[v], c.C, c.grid, shift)[-1, -1, -1, -1]
    got_m = got.clone()
    got_m[-1, -1, -1, -1] = (got[-1, -1, -1, -1].double() - a @ wp[:, 13 * c.C:14 * c.C].t()).to(torch.bfloat16)
    rejects("conv3d: last ragged tile, one tap removed at one voxel", got_m, y, bound)


# ---------------------------------------------------------------------------------------------------- weight gradient
WGRAD_CASES = [
    # kind, (N, H, W) of x, C, Cout, ksplit, Cin (real channels the reduce emits), accumulate
    ("s1", (1, 1, 1), 8, 8, 3, 8, 0),
    ("s1", (2, 5, 3), 72, 72, 1, 72, 0),
    ("s1", (3, 1, 130), 136, 136, 3, 131, 1),
    ("s1", (11, 4, 4), 8, 256, 7, 3, 0),
    ("p1", (1, 1, 1), 136, 256, 1, 136, 1),
    ("p1", (2, 33, 35), 72, 8, 3, 70, 0),
    ("s2", (1, 2, 2), 72, 136, 5, 72, 0),
    ("s2", (2, 10, 6), 136, 72, 3, 136, 1),
    ("s2", (3, 34, 30), 8, 256, 1, 8, 0),
    ("up", (1, 1, 1), 136, 72, 4, 136, 0),
    ("up", (2, 5, 3), 8, 136, 1, 8, 0),
    ("up", (3, 9, 7), 72, 256, 3, 72, 0),
]


def build_wgrad(kind, shp, C, Cout, ksplit, Cin, seed=0):
    P, L = K.plans, K.L
    gen = torch.Generator(device=DEV).manual_seed(seed)
    N, H, W = shp
    Cs, Cys = C + 8, Cout + 8
    X = poisoned(rnd(N, H, W, C, gen=gen), Cs)
    C64 = (C + 63) // 64 * 64
    if kind == "up":
        geoms = [P.geom_up_fwd(N, H, W, Cs, ph, pw) for ph in range(2) for pw in range(2)]
        dyshape = (N, 2 * H, 2 * W)
    else:
        g = P.geom_s2(N, H, W, Cs) if kind == "s2" else P.geom_s1(N, H, W, Cs, 1 if kind == "p1" else 3)
        geoms = [g]
        dyshape = (N, g.Ho, g.Wo)
    for g in geoms:
        g.C = C
    DY = poisoned(rnd(*dyshape, Cout, gen=gen), Cys)
    ntaps = len(geoms[0].taps)
    cols = L.vqb_wgrad_cols(ntaps, C)
    assert cols == ntaps * C64
    if kind == "up":
        ld = 16 * C64
        descs = [P.wgrad_desc(g, Cout, ksplit, dy_view=P.up_dy_view(N, H, W, Cys, p >> 1, p & 1), ld_override=ld,
                              col_offset=p * 4 * C64) for p, g in enumerate(geoms)]
    else:
        ld = cols
        descs = [P.wgrad_desc(geoms[0], Cout, ksplit, dy_view=K.native.dense_view(*dyshape, Cys))]

    def launch():
        part = Guarded(ksplit * Cout * ld, torch.float32)
        for d in descs:
            ok(L.vqb_wgrad_gemm(d, DY.ptr(), X.ptr(), part.ptr(), stream()), f"wgrad_gemm {kind}")
        torch.cuda.synchronize()
        return part

    xf, dyf = X.body.double(), DY.body.double()

    def truth(ccut=0):
        """fp64 dWp[co][p*4*C64 + slot*C64 + c] (c < C) and the same on absolute values, from the descriptors."""
        ref = torch.zeros(Cout, len(geoms) * ntaps, C, device=DEV, dtype=torch.float64)
        S = torch.zeros_like(ref)
        for p, (g, d) in enumerate(zip(geoms, descs)):
            dv = d.dy_view
            grid = (g.N, g.Ho, g.Wo)
            dy = gather(dyf, dv.offset, (dv.Nv, dv.Hv, dv.Wv), (dv.sn, dv.sh, dv.sw), Cout, grid, (0, 0, 0))
            vw, tp = views2d(g)
            for t, (v, shift) in enumerate(tp):
                a = gather(xf, *vw[v], C, grid, shift)
                if ccut:
                    a[..., C - ccut:] = 0
                ref[:, p * ntaps + t] = dy.reshape(-1, Cout).t() @ a.reshape(-1, C)
                S[:, p * ntaps + t] = dy.abs().reshape(-1, Cout).t() @ a.abs().reshape(-1, C)
        return ref, S

    return types.SimpleNamespace(launch=launch, truth=truth, geoms=geoms, descs=descs, ld=ld, C64=C64, ntaps=ntaps,
                                 cols=cols, xf=xf, dyf=dyf, X=X, DY=DY)


def partial_view(c, part, ksplit, Cout):
    """[ksplit][Cout][slots][C64] view of the partial buffer (all launches)."""
    return part.body.view(ksplit, Cout, c.ld)[:, :, :len(c.geoms) * c.cols].reshape(ksplit, Cout, -1, c.C64)


@pytest.mark.parametrize("kind,shp,C,Cout,ksplit,Cin,acc", WGRAD_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_wgrad_bounds(kind, shp, C, Cout, ksplit, Cin, acc):
    P, L = K.plans, K.L
    c = build_wgrad(kind, shp, C, Cout, ksplit, Cin)
    part = c.launch()
    name = f"wgrad {kind} {shp} C={C} Cout={Cout} ksplit={ksplit}"
    written = torch.cat([strided_index(d.col_offset, (ksplit, Cout, c.cols), (Cout * c.ld, c.ld, 1)).reshape(-1)
                         for d in c.descs])
    check_stores(part, written, name + " partial stores")
    pv = partial_view(c, part, ksplit, Cout)
    ref, S = c.truth()
    tau = TAU["wgrad"]
    check(name + " partial", pv.double().sum(0)[:, :, :C], ref, U_F32 * ref.abs() + tau * S,
          acc=(U_F32 * ref.abs(), tau * S))
    if c.C64 > C:  # the C64 padding columns read TMA zero fill only
        check(name + " partial C64 padding columns", pv[:, :, :, C:], torch.zeros_like(pv[:, :, :, C:]), 0.0)
    check_bits(name + " partial", part.bits(), c.launch().bits())
    # split reduction to OIHW
    if kind == "up":
        T = 9
        masks = []
        for g in c.geoms:
            masks += g.tapmask
        tm = torch.tensor(masks, device=DEV, dtype=torch.int32)
        sel = torch.tensor([[(m >> t) & 1 for t in range(T)] for m in masks], device=DEV, dtype=torch.float64)
    else:
        T = 9 if kind in ("s1", "s2") else 1
        tm = torch.tensor(c.geoms[0].tapmap, device=DEV, dtype=torch.int32)
        sel = F.one_hot(tm.long(), T).double()
    gref = torch.einsum("osc,st->oct", ref[:, :, :Cin], sel)
    gS = torch.einsum("osc,st->oct", S[:, :, :Cin], sel)
    grad = Guarded(Cout * Cin * T, torch.float32)
    g0 = None
    if acc:
        g0 = torch.randn(Cout * Cin * T, device=DEV)
        grad.body.copy_(g0)
    nslots = len(c.geoms) * c.ntaps

    def reduce(gbuf):
        if kind == "up":
            ok(L.vqb_wgrad_reduce_fold(part.ptr(), gbuf.ptr(), ksplit, Cout, Cout, Cin, T, nslots, c.C64, tm.data_ptr(),
                                       stream()), "wgrad_reduce_fold")
        else:
            ok(L.vqb_wgrad_reduce(part.ptr(), gbuf.ptr(), ksplit, Cout, Cout, Cin, T, nslots, c.C64, tm.data_ptr(),
                                  acc, stream()), "wgrad_reduce")
        torch.cuda.synchronize()

    reduce(grad)
    check_stores(grad, torch.arange(grad.n, device=DEV), name + " reduce stores")
    got = grad.body.view(Cout, Cin, T)
    psum = partial_view(c, part, ksplit, Cout).double().abs().sum(0)[:, :, :Cin]  # fp32 split sums
    b = U_F32 * gref.abs() + tau * gS + ksplit * U_F32 * torch.einsum("osc,st->oct", psum, sel)
    if acc:
        g0v = g0.double().view(Cout, Cin, T)
        check(name + " reduce accumulate=1", got, g0v + gref, b + U_F32 * (g0v.abs() + gref.abs()))
    else:
        check(name + " reduce", got, gref, b)
        grad2 = Guarded(Cout * Cin * T, torch.float32)
        reduce(grad2)
        check_bits(name + " reduce", grad.bits(), grad2.bits())


def test_wgrad_fold_matches_upsampled_conv():
    """The folded up-sampling weight gradient (4 launches through ld_override / col_offset + vqb_wgrad_reduce_fold)
    equals the fp64 weight gradient of F.conv2d(F.interpolate(x, 2), w, padding=1)."""
    L = K.L
    N, h, w, C, Cout, ksplit = 2, 5, 3, 72, 136, 3
    c = build_wgrad("up", (N, h, w), C, Cout, ksplit, C, seed=11)
    part = c.launch()
    masks = []
    for g in c.geoms:
        masks += g.tapmask
    tm = torch.tensor(masks, device=DEV, dtype=torch.int32)
    grad = Guarded(Cout * C * 9, torch.float32)
    ok(L.vqb_wgrad_reduce_fold(part.ptr(), grad.ptr(), ksplit, Cout, Cout, C, 9, 16, c.C64, tm.data_ptr(), stream()),
       "wgrad_reduce_fold")
    torch.cuda.synchronize()
    x = c.X.body.view(N, h, w, C + 8)[..., :C].double().permute(0, 3, 1, 2)
    dy = c.DY.body.view(N, 2 * h, 2 * w, Cout + 8)[..., :Cout].double().permute(0, 3, 1, 2)

    def dW(xx, gy):
        wr = torch.zeros(Cout, C, 3, 3, device=DEV, dtype=torch.float64, requires_grad=True)
        y = F.conv2d(F.interpolate(xx, scale_factor=2.0, mode="nearest"), wr, padding=1)
        return torch.autograd.grad(y, wr, gy)[0]

    ref, S = dW(x, dy), dW(x.abs(), dy.abs())
    check(f"wgrad folded up-sampling N={N} {h}x{w} C={C} Cout={Cout} vs fp64 interpolate+conv2d",
          grad.body.view(Cout, C, 3, 3), ref, U_F32 * ref.abs() + TAU["wgrad"] * S)


def test_wgrad_mutations_rejected():
    c = build_wgrad("s1", (3, 1, 130), 72, 136, 3, 72, seed=13)
    part = c.launch()
    ref, S = c.truth()
    tau = TAU["wgrad"]
    got = partial_view(c, part, 3, 136).double().sum(0)[:, :, :72]
    bound = U_F32 * ref.abs() + tau * S
    check("wgrad s1 (3,1,130) C=72 Cout=136 (mutation base)", got, ref, bound)
    g_m = got.clone()
    g_m[135, 4] = 0
    rejects("wgrad: tap 4 of the last output channel zeroed", g_m, ref, bound)
    ref_m, S_m = c.truth(ccut=8)
    rejects("wgrad: reference without the last 8 channels of the last K-chunk", got, ref_m,
            U_F32 * ref_m.abs() + tau * S_m)
    # remove the last pixel's (ragged last box) contribution of tap 4 to element (co, 4, c)
    dy_last = c.DY.body.view(3, 1, 130, 144)[2, 0, 129, 135].double()
    x_last = c.X.body.view(3, 1, 130, 80)[2, 0, 129, :72].double()
    g_m = got.clone()
    g_m[135, 4] -= dy_last * x_last
    rejects("wgrad: last ragged pixel box, one tap removed at one pixel", g_m, ref, bound)


# ---------------------------------------------------------------------------------------------------- attention
ATTN_CASES = [
    # T, heads, N, q scale, max key in the ragged tail, q = 0
    (1, 1, 1, 0.5, False, False),
    (2, 3, 3, 3.0, True, False),
    (63, 8, 1, 0.5, True, False),
    (64, 1, 3, 3.0, False, False),
    (65, 3, 1, 3.0, True, False),
    (65, 3, 3, 1.0, False, True),
    (127, 8, 3, 0.5, True, False),
    (129, 1, 1, 3.0, True, False),
    (1000, 3, 3, 0.5, True, False),
    (4097, 1, 1, 3.0, True, False),
]
ATTN_HD32_CASES = [(1, 1, 1, 0.5, False, False), (65, 3, 3, 3.0, True, False), (129, 8, 1, 0.5, True, False),
                   (1000, 1, 3, 3.0, True, False), (4097, 1, 1, 0.5, True, False)]


def attn_inputs(T, heads, N, qs, tail_max, qzero, hd, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    C = heads * hd
    q = torch.randn(N, T, heads, hd, device=DEV, generator=gen) * qs
    k = torch.randn(N, T, heads, hd, device=DEV, generator=gen)
    v = torch.randn(N, T, heads, hd, device=DEV, generator=gen)
    if tail_max:  # every query's largest logit is the last key (last, ragged key tile): the online-softmax rescale
        u = torch.randn(N, 1, heads, hd, device=DEV, generator=gen)
        q = q + u
        k[:, -1] = 3 * u[:, 0] / qs
    if qzero:
        q.zero_()
    qkv = torch.cat([q.reshape(N, T, C), k.reshape(N, T, C), v.reshape(N, T, C)], -1).to(torch.bfloat16)
    return qkv, C


def attn_truth(qkv, heads, hd, scale, swap=None):
    N, T, C3 = qkv.shape
    C = C3 // 3
    x = qkv.double().view(N, T, 3, heads, hd).permute(2, 0, 3, 1, 4)  # [3][N][h][T][hd]
    q, k, v = x[0], x[1], x[2]
    if swap is not None:
        k = k.clone()
        k[:, :, [swap[0], swap[1]]] = k[:, :, [swap[1], swap[0]]]
    s = (q @ k.transpose(-1, -2)) * scale
    lse = torch.logsumexp(s, -1)
    p = torch.softmax(s, -1)
    o = p @ v
    oa = p @ v.abs()
    qk = q.abs() @ k.abs().transpose(-1, -2) * scale
    return o, oa, lse, qk.amax(-1)


def attn_check_fwd(name, out, lse, qkv, heads, hd, scale, swap=None, mutation=False):
    N, T, _ = qkv.shape
    C = heads * hd
    o, oa, lse64, qkmax = attn_truth(qkv, heads, hd, scale, swap)
    got = out.body.view(N, T, heads, hd).permute(0, 2, 1, 3)
    bound = U_BF16 * o.abs() + U_BF16 * oa
    if mutation:
        rejects(name, got, o, bound)
        return
    check(name + " out", got, o, bound)
    # lse: fp32 logit accumulation over hd products, __expf/__logf, fp32 running sum over T keys
    lb = 2.0 ** -18 * (1 + qkmax + lse64.abs()) + T * U_F32
    check(name + " lse", lse.body.view(N, heads, T), lse64, lb)


def attn_run_fwd(qkv, C, hd):
    N, T, _ = qkv.shape
    heads = C // hd
    Q = Guarded(qkv.numel(), torch.bfloat16, poison="nan")
    Q.body.copy_(qkv.reshape(-1))
    out = Guarded(N * T * C, torch.bfloat16)
    lse = Guarded(N * heads * T, torch.float32)
    if hd == 64:
        ok(K.L.vqb_attn_fwd(Q.ptr(), out.ptr(), lse.ptr(), N, T, C, stream()), "attn_fwd")
    else:
        ok(K.L.vqb_attn_fwd_hd(Q.ptr(), out.ptr(), lse.ptr(), N, T, C, hd, stream()), "attn_fwd_hd")
    torch.cuda.synchronize()
    return Q, out, lse


def rowwise(name, got, ref, inherent):
    """L2 error per (n, head, token) row <= 2^-6 of the row's fp64 norm + the L2 norm of `inherent` over that row."""
    e = (got.double() - ref).norm(dim=-1)
    return check(name, e, torch.zeros_like(e), 2.0 ** -6 * ref.norm(dim=-1) + inherent.norm(dim=-1))


def attn_bwd_inherent(qkv, o_bf16, dout, heads, hd, scale):
    """Per-element error terms of dq, dk, dv ([N][T][heads][hd] each) that the flash-attention backward inherits:
    D = rowsum(dO * O) is formed from the bf16 output O (|dD| <= sum |dO| (2^-8 |O| + 2^-8 P|V|), the forward bound),
    and P and dS are rounded to bf16 before their second GEMM (2^-8 of |P| |dO|, |dS| |K|, |dS|^T |Q|). When the softmax
    is nearly one-hot, dq and dk are differences of nearly equal terms and these dominate the row norm."""
    N, T, _ = qkv.shape
    x = qkv.double().view(N, T, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    dO = dout.double().view(N, T, heads, hd).transpose(1, 2)
    O = o_bf16.double().view(N, T, heads, hd).transpose(1, 2)
    P = torch.softmax((q @ k.transpose(-1, -2)) * scale, -1)
    dD = (dO.abs() * (U_BF16 * O.abs() + U_BF16 * (P @ v.abs()))).sum(-1, keepdim=True)  # [N][h][T][1]
    dP = dO @ v.transpose(-1, -2)
    dS = P * (dP - (dO * O).sum(-1, keepdim=True))
    e_dq = scale * (dD * (P @ k.abs()) + U_BF16 * (dS.abs() @ k.abs()))
    e_dk = scale * ((P * dD).transpose(-1, -2) @ q.abs() + U_BF16 * (dS.abs().transpose(-1, -2) @ q.abs()))
    e_dv = U_BF16 * (P.transpose(-1, -2) @ dO.abs())
    return [t.transpose(1, 2) for t in (e_dq, e_dk, e_dv)]


@pytest.mark.parametrize("T,heads,N,qs,tail,qzero", ATTN_CASES, ids=lambda v: str(v))
def test_attention_hd64_bounds(T, heads, N, qs, tail, qzero):
    hd, scale = 64, 0.125
    qkv, C = attn_inputs(T, heads, N, qs, tail, qzero, hd, seed=T + heads)
    Q, out, lse = attn_run_fwd(qkv, C, hd)
    name = f"attn hd=64 T={T} heads={heads} N={N} qscale={qs}{' tail-max' if tail else ''}{' q=0' if qzero else ''}"
    check_stores(out, torch.arange(out.n, device=DEV), name + " out stores")
    check_stores(lse, torch.arange(lse.n, device=DEV), name + " lse stores")
    attn_check_fwd(name, out, lse, qkv, heads, hd, scale)
    if qzero:
        mean_v = qkv.double()[..., 2 * C:].mean(1).view(N, 1, heads, hd).permute(0, 2, 1, 3)
        check(name + " out = mean(v)", out.body.view(N, T, heads, hd).permute(0, 2, 1, 3),
              mean_v.expand(N, heads, T, hd), U_BF16 * mean_v.abs() + 2.0 ** -16)
    _, out2, lse2 = attn_run_fwd(qkv, C, hd)
    check_bits(name + " fwd", out.bits(), out2.bits())
    check_bits(name + " lse", lse.bits(), lse2.bits())
    # backward
    gen = torch.Generator(device=DEV).manual_seed(T)
    dout = rnd(N, T, C, gen=gen)
    DO = Guarded(dout.numel(), torch.bfloat16, poison="nan")
    DO.body.copy_(dout.reshape(-1))

    def bwd():
        dvec = Guarded(N * heads * T, torch.float32)
        dq = Guarded(N * T * 3 * C, torch.bfloat16)
        ok(K.L.vqb_attn_bwd(Q.ptr(), out.ptr(), DO.ptr(), lse.ptr(), dvec.ptr(), dq.ptr(), N, T, C, stream()),
           "attn_bwd")
        torch.cuda.synchronize()
        return dvec, dq

    dvec, dq = bwd()
    check_stores(dq, torch.arange(dq.n, device=DEV), name + " dqkv stores")
    check_stores(dvec, torch.arange(dvec.n, device=DEV), name + " dvec stores")
    x = qkv.double().view(N, T, 3, heads, hd).requires_grad_(True)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))
    o = torch.softmax((q @ k.transpose(-1, -2)) * scale, -1) @ v
    (gx,) = torch.autograd.grad(o, x, dout.double().view(N, T, heads, hd).transpose(1, 2))
    got = dq.body.view(N, T, 3, heads, hd)
    inh = attn_bwd_inherent(qkv, out.body.view(N, T, C), dout, heads, hd, scale)
    for i, nm in enumerate(("dq", "dk", "dv")):
        rowwise(f"{name} {nm} rows", got[:, :, i], gx[:, :, i], inh[i])
    _, dq2 = bwd()
    check_bits(name + " bwd", dq.bits(), dq2.bits())


@pytest.mark.parametrize("T,heads,N,qs,tail,qzero", ATTN_HD32_CASES, ids=lambda v: str(v))
def test_attention_hd32_bounds(T, heads, N, qs, tail, qzero):
    hd = 32
    qkv, C = attn_inputs(T, heads, N, qs, tail, qzero, hd, seed=T + 7)
    Q, out, lse = attn_run_fwd(qkv, C, hd)
    name = f"attn hd=32 T={T} heads={heads} N={N} qscale={qs}{' tail-max' if tail else ''}"
    check_stores(out, torch.arange(out.n, device=DEV), name + " out stores")
    check_stores(lse, torch.arange(lse.n, device=DEV), name + " lse stores")
    attn_check_fwd(name, out, lse, qkv, heads, hd, 32 ** -0.5)
    _, out2, _ = attn_run_fwd(qkv, C, hd)
    check_bits(name + " fwd", out.bits(), out2.bits())


def test_attention_mutation_rejected():
    """A reference with two keys of the ragged tail swapped (k rows only) is rejected."""
    T, heads, N = 127, 3, 1
    qkv, C = attn_inputs(T, heads, N, 3.0, False, False, 64, seed=21)
    _, out, lse = attn_run_fwd(qkv, C, 64)
    attn_check_fwd("attn T=127 (mutation base)", out, lse, qkv, heads, 64, 0.125)
    attn_check_fwd("attention: reference with keys 125 and 126 of the ragged tail swapped", out, lse, qkv, heads, 64,
                   0.125, swap=(125, 126), mutation=True)


# ---------------------------------------------------------------------------------------------------- GroupNorm
GN_SHAPES = [(1, 1, 64), (2, 7, 32), (3, 1000, 96), (2, 5, 2048), (1, 3 * 2 ** 16 + 5, 64), (1, 48 * 32 * 32, 256)]
GN_FWD_CASES = [(s, silu, r) for i, s in enumerate(GN_SHAPES) for silu, r in (((i + 1) % 2, (0, 5, 20)[i % 3]),
                                                                               (i % 2, (20, 0, 5)[i % 3]))]
G32 = 32
EPS = 1e-6


def gn_inputs(N, HW, C, ratio, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = ((torch.randn(N, HW, C, device=DEV, generator=gen) + ratio) * 2).to(torch.bfloat16)
    gamma = torch.randn(C, device=DEV, generator=gen) * 0.5 + 1
    beta = torch.randn(C, device=DEV, generator=gen) * 0.2
    return x, gamma, beta, gen


def gn_stats64(x64, G, drop_last=False, bessel=False):
    N, HW, C = x64.shape
    xg = x64.view(N, HW, G, C // G)
    if drop_last:
        xg = xg[:, :-1]
    m = xg.shape[1] * xg.shape[3]
    mean = xg.sum((1, 3)) / m
    var = ((xg - mean[:, None, :, None]) ** 2).sum((1, 3)) / (m - 1 if bessel else m)
    return mean, var


def gn_fwd_truth(x, gamma, beta, silu, mean, var):
    N, HW, C = x.shape
    grp = torch.arange(C, device=DEV) // (C // G32)
    rstd = 1 / torch.sqrt(var + EPS)
    mc, rc = mean[:, grp].view(N, 1, C), rstd[:, grp].view(N, 1, C)
    x64 = x.double()
    u = (x64 - mc) * rc * gamma.double() + beta.double()
    y = u * torch.sigmoid(u) if silu else u
    # statistics bounds (fp32 partial sums combined in double) and their effect on y
    sd = var.sqrt()
    dmean = 2.0 ** -14 * (mean.abs() + sd)
    drstd = 2.0 ** -14 * (1 + mean ** 2 / (var + EPS)) * rstd
    stat = gamma.double().abs() * (dmean[:, grp].view(N, 1, C) * rc + (x64 - mc).abs() * drstd[:, grp].view(N, 1, C))
    bound = U_BF16 * y.abs() + (2.0 ** -11 * u.abs() if silu else 0) + 1.1 * stat
    return y, bound, rstd, dmean, drstd


@pytest.mark.parametrize("shape,silu,ratio", GN_FWD_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_gn_silu_fwd_bounds(shape, silu, ratio):
    N, HW, C = shape
    x, gamma, beta, _ = gn_inputs(N, HW, C, ratio, seed=HW + C)
    X = Guarded(x.numel(), torch.bfloat16, poison="nan")
    X.body.copy_(x.reshape(-1))
    name = f"gn_silu_fwd N={N} HW={HW} C={C} silu={silu} mean/std={ratio}"
    mean, var = gn_stats64(x.double(), G32)
    y64, bound, rstd, dmean, drstd = gn_fwd_truth(x, gamma, beta, silu, mean, var)

    def run():
        y = Guarded(x.numel(), torch.bfloat16)
        mr = Guarded(N * G32 * 2, torch.float32)
        ws = torch.empty(N * C * 2, device=DEV, dtype=torch.float64)
        ok(K.L.vqb_gn_silu_fwd(X.ptr(), y.ptr(), gamma.data_ptr(), beta.data_ptr(), mr.ptr(), ws.data_ptr(), N, HW, C,
                               G32, EPS, silu, stream()), "gn_silu_fwd")
        torch.cuda.synchronize()
        return y, mr

    y, mr = run()
    check_stores(y, torch.arange(y.n, device=DEV), name + " stores")
    check_stores(mr, torch.arange(mr.n, device=DEV), name + " mr stores")
    mrv = mr.body.view(N, G32, 2)
    check(name + " mean", mrv[..., 0], mean, dmean)
    check(name + " rstd", mrv[..., 1], rstd, drstd)
    check(name, y.body.view(N, HW, C), y64, bound)
    y2, mr2 = run()
    check_bits(name, y.bits(), y2.bits())
    check_bits(name + " mr", mr.bits(), mr2.bits())
    # the apply pass fed fp64-derived channel sums (the conv-epilogue statistics route)
    x64 = x.double()
    chs = torch.stack([x64.sum(1), (x64 * x64).sum(1)], -1).float().contiguous()
    yp = Guarded(x.numel(), torch.bfloat16)
    mrp = Guarded(N * G32 * 2, torch.float32)
    ok(K.L.vqb_gn_silu_fwd_pre(X.ptr(), yp.ptr(), gamma.data_ptr(), beta.data_ptr(), mrp.ptr(), chs.data_ptr(), N, HW,
                               C, G32, EPS, silu, stream()), "gn_silu_fwd_pre")
    torch.cuda.synchronize()
    check_stores(yp, torch.arange(yp.n, device=DEV), name + " _pre stores")
    check(name + " _pre", yp.body.view(N, HW, C), y64, bound)


GN_BWD_CASES = [
    # shape, silu, add, dx_colsum, dx aliases dy
    ((1, 1, 64), 1, False, True, False),
    ((2, 7, 32), 0, True, False, True),
    ((3, 1000, 96), 1, True, True, False),
    ((3, 1000, 96), 1, False, False, False),
    ((2, 5, 2048), 0, False, True, True),
    ((2, 5, 2048), 1, True, False, False),
    ((1, 3 * 2 ** 16 + 5, 64), 1, False, True, True),
    ((1, 48 * 32 * 32, 256), 1, True, True, False),
    ((1, 48 * 32 * 32, 256), 0, False, False, False),
]


@pytest.mark.parametrize("shape,silu,add,colsum,alias", GN_BWD_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_gn_silu_bwd_bounds(shape, silu, add, colsum, alias):
    N, HW, C = shape
    x, gamma, beta, gen = gn_inputs(N, HW, C, 1.0, seed=HW + C + 1)
    dy = rnd(N, HW, C, gen=gen)
    ad = rnd(N, HW, C, gen=gen) if add else None
    mean, var = gn_stats64(x.double(), G32)
    rstd = 1 / torch.sqrt(var + EPS)
    mr = torch.stack([mean, rstd], -1).float().contiguous()  # the kernel reads the fp32-rounded statistics
    meanf, rstdf = mr[..., 0].double(), mr[..., 1].double()
    grp = torch.arange(C, device=DEV) // (C // G32)
    x64, dy64 = x.double(), dy.double()
    mc, rc = meanf[:, grp].view(N, 1, C), rstdf[:, grp].view(N, 1, C)
    xh = (x64 - mc) * rc
    ga = gamma.double()
    u = xh * ga + beta.double()
    if silu:
        sg = torch.sigmoid(u)
        du = dy64 * sg * (1 + u * (1 - sg))
        edu = 2.0 ** -11 * dy64.abs() * (1 + u.abs())  # MUFU.TANH sigmoid inside silu'
    else:
        du = dy64
        edu = torch.zeros_like(du)
    cpg = C // G32

    def gmean(t):  # per-(n, group) mean over pixels and the group's channels, broadcast back to [N, 1, C]
        return t.view(N, HW, G32, cpg).mean((1, 3))[:, grp].view(N, 1, C)

    g1, g2 = gmean(ga * du), gmean(ga * du * xh)
    dx64 = rc * (ga * du - g1 - xh * g2)
    if add:
        dx64 = dx64 + ad.double()
    e1, e2 = gmean(ga.abs() * edu), gmean(ga.abs() * edu * xh.abs())
    bound = U_BF16 * dx64.abs() + rc * (ga.abs() * edu + e1 + xh.abs() * e2) + \
        2.0 ** -16 * rc * ((ga * du).abs() + g1.abs() + (xh * g2).abs())
    cs64 = torch.stack([du.sum(1), (du * xh).sum(1)], -1)  # [N, C, 2]
    Xg = Guarded(x.numel(), torch.bfloat16, poison="nan")
    Xg.body.copy_(x.reshape(-1))
    Ag = None
    if add:
        Ag = Guarded(x.numel(), torch.bfloat16, poison="nan")
        Ag.body.copy_(ad.reshape(-1))
    name = f"gn_silu_bwd N={N} HW={HW} C={C} silu={silu} add={add} colsum={colsum} dx-aliases-dy={alias}"
    DY = Guarded(x.numel(), torch.bfloat16, poison="nan")
    DY.body.copy_(dy.reshape(-1))
    dx = DY if alias else Guarded(x.numel(), torch.bfloat16)
    dg = Guarded(C, torch.float32)
    db = Guarded(C, torch.float32)
    cs_out = Guarded(C, torch.float32) if colsum else None
    ws = torch.empty(N * C * 2 + N * G32 * 2, device=DEV, dtype=torch.float32)
    ok(K.L.vqb_gn_silu_bwd(Xg.ptr(), DY.ptr(), Ag.ptr() if Ag else 0, dx.ptr(), gamma.data_ptr(), beta.data_ptr(),
                           mr.data_ptr(), dg.ptr(), db.ptr(), ws.data_ptr(), N, HW, C, G32, silu,
                           cs_out.ptr() if cs_out else 0, stream()), "gn_silu_bwd")
    torch.cuda.synchronize()
    if not alias:
        check_stores(dx, torch.arange(dx.n, device=DEV), name + " dx stores")
    else:
        assert (DY.buf[:DY.g].isnan().all() and DY.buf[DY.g + DY.n:].isnan().all()), name + ": guard band written"
    got = dx.body.view(N, HW, C)
    check(name + " dx", got, dx64, bound)
    for G_, nm, ref, w in ((db, "dbeta", cs64[..., 0].sum(0), edu), (dg, "dgamma", cs64[..., 1].sum(0),
                                                                     edu * xh.abs())):
        check_stores(G_, torch.arange(C, device=DEV), f"{name} {nm} stores")
        terms = (du.abs() if nm == "dbeta" else (du * xh).abs())
        check(f"{name} {nm}", G_.body, ref, w.sum((0, 1)) + 2.0 ** -14 * terms.sum((0, 1)))
    if colsum:
        check_stores(cs_out, torch.arange(C, device=DEV), name + " dx_colsum stores")
        v = got.double()
        check(name + " dx_colsum (vs fp64 sum of the bf16 dx written)", cs_out.body, v.sum((0, 1)),
              2.0 ** -14 * v.abs().sum((0, 1)))


def test_gn_mutations_rejected():
    """The GroupNorm checker rejects references with the unbiased variance or a statistic that skipped one pixel."""
    N, HW, C = 2, 7, 32
    x, gamma, beta, _ = gn_inputs(N, HW, C, 5, seed=31)
    y = torch.empty_like(x)
    mr = torch.empty(N, G32, 2, device=DEV)
    ws = torch.empty(N * C * 2, device=DEV, dtype=torch.float64)
    ok(K.L.vqb_gn_silu_fwd(x.data_ptr(), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(), mr.data_ptr(), ws.data_ptr(),
                           N, HW, C, G32, EPS, 1, stream()), "gn_silu_fwd")
    torch.cuda.synchronize()
    mean, var = gn_stats64(x.double(), G32)
    y64, bound = gn_fwd_truth(x, gamma, beta, 1, mean, var)[:2]
    check("gn (2,7,32) (mutation base)", y, y64, bound)
    mean_b, var_b = gn_stats64(x.double(), G32, bessel=True)
    y_b, bound_b = gn_fwd_truth(x, gamma, beta, 1, mean_b, var_b)[:2]
    rejects("gn: reference with the unbiased (Bessel) variance", y, y_b, bound_b)
    mean_d, var_d = gn_stats64(x.double(), G32, drop_last=True)
    y_d, bound_d = gn_fwd_truth(x, gamma, beta, 1, mean_d, var_d)[:2]
    rejects("gn: reference statistics without the last pixel", y, y_d, bound_d)


# ---------------------------------------------------------------------------------------------------- layout, pack
@pytest.mark.parametrize("Cpad", [8, 16])
def test_layout_conversions(Cpad):
    L = K.L
    gen = torch.Generator(device=DEV).manual_seed(Cpad)
    N, C, H, W = 2, 3, 5, 130
    shift = torch.tensor([-0.03, -0.088, -0.188], device=DEV)
    isc = 1.0 / torch.tensor([0.458, 0.448, 0.45], device=DEV)
    x32 = torch.randn(N, C, H, W, device=DEV, generator=gen)
    x16 = x32.to(torch.bfloat16)
    for src, fn in ((x32, "vqb_nchw_to_nhwc"), (x16, "vqb_nchw_to_nhwc_bf16")):
        Xg = Guarded(src.numel(), src.dtype, poison="nan")
        Xg.body.copy_(src.reshape(-1))
        for scaled in (False, True):
            def run():
                y = Guarded(N * H * W * Cpad, torch.bfloat16)
                ok(getattr(L, fn)(Xg.ptr(), y.ptr(), N, C, H, W, Cpad, shift.data_ptr() if scaled else 0,
                                  isc.data_ptr() if scaled else 0, stream()), fn)
                torch.cuda.synchronize()
                return y
            y = run()
            name = f"{fn} C=3 Cpad={Cpad} {'scaled' if scaled else 'plain'}"
            check_stores(y, torch.arange(y.n, device=DEV), name + " stores")
            got = y.body.view(N, H, W, Cpad)
            check(name + " pad channels are zero", got[..., C:], torch.zeros_like(got[..., C:]), 0.0)
            if scaled:
                ref = ((src.float() - shift.view(1, C, 1, 1)) * isc.view(1, C, 1, 1)).permute(0, 2, 3, 1)
                check(name, got[..., :C], ref.double(), bf16_ulp(ref))
            else:
                check(name + " (exact)", got[..., :C], src.permute(0, 2, 3, 1).to(torch.bfloat16), 0.0)
            check_bits(name, y.bits(), run().bits())
    # into the interior of a framed buffer: the frame is not touched
    for src, fn in ((x32, "vqb_nchw_to_nhwc_pad"), (x16, "vqb_nchw_to_nhwc_pad_bf16")):
        Xg = Guarded(src.numel(), src.dtype, poison="nan")
        Xg.body.copy_(src.reshape(-1))
        y = Guarded(N * (H + 2) * (W + 2) * Cpad, torch.bfloat16)
        ok(getattr(L, fn)(Xg.ptr(), y.ptr(), N, C, H, W, Cpad, 1, 0, 0, stream()), fn)
        torch.cuda.synchronize()
        name = f"{fn} C=3 Cpad={Cpad} pad=1"
        inner = strided_index(((W + 2) + 1) * Cpad, (N, H, W, Cpad),
                              ((H + 2) * (W + 2) * Cpad, (W + 2) * Cpad, Cpad, 1))
        check_stores(y, inner, name + " stores (frame untouched)")
        got = y.body[inner]
        check(name + " pad channels are zero", got[..., C:], torch.zeros_like(got[..., C:]), 0.0)
        check(name + " (exact)", got[..., :C], src.permute(0, 2, 3, 1).to(torch.bfloat16), 0.0)
    # NHWC -> NCHW: pad channels and the frame are NaN, so an over-read shows
    g = rnd(N, H, W, C, gen=gen)
    G = poisoned(g, Cpad)
    for scaled in (False, True):
        gx = Guarded(N * C * H * W, torch.float32)
        ok(L.vqb_nhwc_to_nchw(G.ptr(), gx.ptr(), N, C, H, W, Cpad, isc.data_ptr() if scaled else 0, stream()),
           "nhwc_to_nchw")
        torch.cuda.synchronize()
        name = f"vqb_nhwc_to_nchw C=3 Cpad={Cpad} {'scaled' if scaled else 'plain'}"
        check_stores(gx, torch.arange(gx.n, device=DEV), name + " stores")
        ref = g.double().permute(0, 3, 1, 2) * (isc.double().view(1, C, 1, 1) if scaled else 1)
        check(name, gx.body.view(N, C, H, W), ref, 2.0 ** -24 * ref.abs())
    xb = Guarded(N * C * H * W, torch.bfloat16)
    ok(L.vqb_nhwc_to_nchw_bf16(G.ptr(), xb.ptr(), N, C, H, W, Cpad, stream()), "nhwc_to_nchw_bf16")
    torch.cuda.synchronize()
    check_stores(xb, torch.arange(xb.n, device=DEV), "vqb_nhwc_to_nchw_bf16 stores")
    check(f"vqb_nhwc_to_nchw_bf16 C=3 Cpad={Cpad} (exact)", xb.body.view(N, C, H, W), g.permute(0, 3, 1, 2), 0.0)
    xb2 = Guarded(N * C * H * W, torch.bfloat16)
    ok(L.vqb_nhwc_to_nchw_bf16(G.ptr(), xb2.ptr(), N, C, H, W, Cpad, stream()), "nhwc_to_nchw_bf16")
    torch.cuda.synchronize()
    check_bits("vqb_nhwc_to_nchw_bf16", xb.bits(), xb2.bits())
    framed = torch.full((N, H + 2, W + 2, Cpad), float("nan"), device=DEV, dtype=torch.bfloat16)
    framed[:, 1:-1, 1:-1, :C] = g
    Fg = Guarded(framed.numel(), torch.bfloat16, poison="nan")
    Fg.body.copy_(framed.reshape(-1))
    gx = Guarded(N * C * H * W, torch.float32)
    ok(L.vqb_nhwc_to_nchw_pad(Fg.ptr(), gx.ptr(), N, C, H, W, Cpad, 1, isc.data_ptr(), stream()), "nhwc_to_nchw_pad")
    torch.cuda.synchronize()
    check_stores(gx, torch.arange(gx.n, device=DEV), "vqb_nhwc_to_nchw_pad stores")
    ref = g.double().permute(0, 3, 1, 2) * isc.double().view(1, C, 1, 1)
    check(f"vqb_nhwc_to_nchw_pad C=3 Cpad={Cpad} scaled (NaN frame, NaN pad channels)", gx.body.view(N, C, H, W), ref,
          2.0 ** -24 * ref.abs())


PACK_CASES = [(64, 48, 9, 0), (64, 48, 9, 1), (5, 136, 1, 0), (128, 3, 9, 1), (72, 24, 27, 0), (16, 8, 27, 1)]


@pytest.mark.parametrize("Cout,Cin,T,tr", PACK_CASES, ids=lambda v: str(v))
def test_pack_weights(Cout, Cin, T, tr):
    L = K.L
    gen = torch.Generator(device=DEV).manual_seed(Cout + Cin + T)
    w32 = torch.randn(Cout, Cin, T, device=DEV, generator=gen)
    w16 = w32.to(torch.bfloat16)
    R, Kk = (Cin, Cout) if tr else (Cout, Cin)
    Kpad = (Kk + 7) // 8 * 8 + 8
    tapmap = list(range(T))[::-1] if tr else list(range(T))
    tm = torch.tensor(tapmap, device=DEV, dtype=torch.int32)
    for w, fn in ((w32, "vqb_pack_weights"), (w16, "vqb_pack_weights_bf16")):
        W_ = Guarded(w.numel(), w.dtype, poison="nan")
        W_.body.copy_(w.reshape(-1))

        def run():
            out = Guarded(R * T * Kpad, torch.bfloat16)
            ok(getattr(L, fn)(W_.ptr(), out.ptr(), Cout, Cin, T, T, tm.data_ptr(), tr, Kpad, stream()), fn)
            torch.cuda.synchronize()
            return out
        out = run()
        name = f"{fn} Cout={Cout} Cin={Cin} T={T} transpose={tr}"
        check_stores(out, torch.arange(out.n, device=DEV), name + " stores")
        src = w.to(torch.bfloat16)[:, :, tapmap]  # [Cout, Cin, slot]
        m = src.permute(1, 2, 0) if tr else src.permute(0, 2, 1)
        ref = torch.zeros(R, T, Kpad, device=DEV, dtype=torch.bfloat16)
        ref[:, :, :Kk] = m
        check(name + " (exact)", out.body.view(R, T, Kpad), ref, 0.0)
        check_bits(name, out.bits(), run().bits())
    # folded slots: bit masks of taps summed in fp32 and rounded once: within one bf16 ulp of the fp64 sum
    masks = [(1 << (s % T)) | (1 << ((3 * s + 1) % T)) | (1 << ((5 * s + 2) % T)) for s in range(min(T, 8))]
    mk = torch.tensor(masks, device=DEV, dtype=torch.int32)
    sel = torch.tensor([[(mm >> t) & 1 for t in range(T)] for mm in masks], device=DEV, dtype=torch.float64)
    for w, fn in ((w32, "vqb_pack_weights_fold"), (w16, "vqb_pack_weights_fold_bf16")):
        W_ = Guarded(w.numel(), w.dtype, poison="nan")
        W_.body.copy_(w.reshape(-1))
        out = Guarded(R * len(masks) * Kpad, torch.bfloat16)
        ok(getattr(L, fn)(W_.ptr(), out.ptr(), Cout, Cin, T, len(masks), mk.data_ptr(), tr, Kpad, stream()), fn)
        torch.cuda.synchronize()
        name = f"{fn} Cout={Cout} Cin={Cin} T={T} transpose={tr}"
        check_stores(out, torch.arange(out.n, device=DEV), name + " stores")
        s64 = torch.einsum("oit,st->ois", w.double(), sel)
        m = s64.permute(1, 2, 0) if tr else s64.permute(0, 2, 1)
        ref = torch.zeros(R, len(masks), Kpad, device=DEV, dtype=torch.float64)
        ref[:, :, :Kk] = m
        # one ulp, plus the fp32 summation error of an fp32 master (|sum| << sum |w| under cancellation)
        asum = torch.einsum("oit,st->ois", w.double().abs(), sel)
        asum = asum.permute(1, 2, 0) if tr else asum.permute(0, 2, 1)
        tol = torch.zeros_like(ref)
        tol[:, :, :Kk] = bf16_ulp(ref[:, :, :Kk]) + (2.0 ** -22 if w.dtype == torch.float32 else 0.0) * asum
        check(name + " (one bf16 ulp of the fp64 tap sum)", out.body.view(R, len(masks), Kpad), ref, tol)


def test_pack_weights_multi():
    """One launch, mixed fp32 / bf16 masters, plain and folded jobs: exact re-layout / one ulp of the fp64 tap sum."""
    L = K.L
    gen = torch.Generator(device=DEV).manual_seed(41)
    specs = [(64, 48, 9, 0, 0, torch.float32), (24, 136, 9, 1, 0, torch.bfloat16), (72, 8, 9, 0, 1, torch.bfloat16),
             (8, 3, 1, 0, 0, torch.float32)]
    jobs, outs, keep = [], [], []
    first = 0
    for (Cout, Cin, T, tr, fold, dt) in specs:
        w = torch.randn(Cout, Cin, T, device=DEV, generator=gen).to(dt)
        R, Kk = (Cin, Cout) if tr else (Cout, Cin)
        Kpad = (Kk + 7) // 8 * 8
        if fold:
            tapmap = [3, 6, 5, 9 | 2, 511]
        else:
            tapmap = list(range(T))[::-1] if tr else list(range(T))
        ns = len(tapmap)
        tm = torch.tensor(tapmap, device=DEV, dtype=torch.int32)
        out = Guarded(R * ns * Kpad, torch.bfloat16)
        jobs.append(K.native.VqbPackJob(w=w.data_ptr(), out=out.ptr(), tapmap=tm.data_ptr(), Cout=Cout, Cin=Cin, T=T,
                                        nslots=ns, transpose=tr, Kpad=Kpad, fold=fold, sg=ns, ld_g=0, ld_r=ns * Kpad,
                                        first_block=first, w_bf16=1 if dt == torch.bfloat16 else 0))
        first += -(-R // 8) * -(-Kpad // 64)
        outs.append((out, w, tapmap, R, Kk, Kpad, tr, fold))
        keep += [w, tm]
    import ctypes
    arr = (K.native.VqbPackJob * len(jobs))(*jobs)
    jt = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(DEV)
    ok(L.vqb_pack_weights_multi(jt.data_ptr(), len(jobs), first, stream()), "pack_weights_multi")
    torch.cuda.synchronize()
    assert ctypes.sizeof(K.native.VqbPackJob) * len(jobs) == jt.numel()
    for (out, w, tapmap, R, Kk, Kpad, tr, fold) in outs:
        name = f"vqb_pack_weights_multi {tuple(w.shape)} {w.dtype} transpose={tr} fold={fold}"
        check_stores(out, torch.arange(out.n, device=DEV), name + " stores")
        T = w.shape[2]
        if fold:
            sel = torch.tensor([[(m >> t) & 1 for t in range(T)] for m in tapmap], device=DEV, dtype=torch.float64)
            s = torch.einsum("oit,st->ois", w.double(), sel)
        else:
            s = w.to(torch.bfloat16)[:, :, tapmap].double()
        m = s.permute(1, 2, 0) if tr else s.permute(0, 2, 1)
        ref = torch.zeros(R, len(tapmap), Kpad, device=DEV, dtype=torch.float64)
        ref[:, :, :Kk] = m
        tol = torch.where(ref == 0, torch.zeros_like(ref), bf16_ulp(ref)) if fold else 0.0
        check(name, out.body.view(R, len(tapmap), Kpad), ref, tol)


# ---------------------------------------------------------------------------------------------------- small kernels
@pytest.mark.parametrize("bf16", [0, 1])
def test_wavelet_fwd(bf16):
    L = K.L
    gen = torch.Generator(device=DEV).manual_seed(51 + bf16)
    N, C, H, W, Cp = 2, 3, 10, 34, 16
    x = torch.randn(N, C, H, W, device=DEV, generator=gen)
    if bf16:
        x = x.to(torch.bfloat16)
    filt = torch.randn(4, 6, 6, device=DEV, generator=gen) * 0.3
    X = Guarded(x.numel(), x.dtype, poison="nan")
    X.body.copy_(x.reshape(-1))
    y = Guarded(N * (H // 2) * (W // 2) * Cp, torch.bfloat16)
    fn = "vqb_wavelet_fwd_bf16" if bf16 else "vqb_wavelet_fwd"
    ok(getattr(L, fn)(X.ptr(), y.ptr(), filt.data_ptr(), N, C, H, W, Cp, stream()), fn)
    torch.cuda.synchronize()
    name = f"{fn} N={N} C={C} {H}x{W} Cpad={Cp}"
    check_stores(y, torch.arange(y.n, device=DEV), name + " stores")
    xp = F.pad(x.double(), (2, 2, 2, 2))
    wt = filt.double().view(4, 1, 6, 6).repeat(C, 1, 1, 1)
    ref = F.conv2d(xp, wt, stride=2, groups=C).permute(0, 2, 3, 1)  # channel c*4 + band
    S = F.conv2d(xp.abs(), wt.abs(), stride=2, groups=C).permute(0, 2, 3, 1)
    got = y.body.view(N, H // 2, W // 2, Cp)
    check(name, got[..., :4 * C], ref, U_BF16 * ref.abs() + 2.0 ** -20 * S)
    check(name + " pad channels are zero", got[..., 4 * C:], torch.zeros_like(got[..., 4 * C:]), 0.0)


def test_maxpool2_bounds():
    L = K.L
    gen = torch.Generator(device=DEV).manual_seed(61)
    N, C = 2, 24
    # max-pool: ties (first maximum wins), all-negative windows (ReLU gate), add operand
    Ho, Wo = 3, 5
    xm = torch.randn(N, 2 * Ho, 2 * Wo, C, device=DEV, generator=gen).to(torch.bfloat16)
    xm = torch.where(torch.rand(xm.shape, device=DEV, generator=gen) < 0.3, torch.ones_like(xm), xm)  # ties at 1
    xm[0, 0:2, 0:2, :] = -0.5  # a window of equal non-positive values
    XM = poisoned(xm, C)
    yp = Guarded(N * Ho * Wo * C, torch.bfloat16)
    ok(L.vqb_maxpool2_fwd(XM.ptr(), yp.ptr(), N, Ho, Wo, C, stream()), "maxpool2_fwd")
    torch.cuda.synchronize()
    check_stores(yp, torch.arange(yp.n, device=DEV), "maxpool2_fwd stores")
    win = xm.double().view(N, Ho, 2, Wo, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(N, Ho, Wo, C, 4)
    check("maxpool2_fwd (exact)", yp.body.view(N, Ho, Wo, C), win.amax(-1), 0.0)
    first = win.argmax(-1)  # torch.argmax returns the first maximal index
    gdy = rnd(N, Ho, Wo, C, gen=gen)
    GDY = poisoned(gdy, C)
    ad = rnd(N, 2 * Ho, 2 * Wo, C, gen=gen)
    AD = poisoned(ad, C)
    for relu, use_add in ((1, True), (0, False), (1, False)):
        dxm = Guarded(xm.numel(), torch.bfloat16)
        ok(L.vqb_maxpool2_bwd(XM.ptr(), GDY.ptr(), AD.ptr() if use_add else 0, dxm.ptr(), N, Ho, Wo, C, relu,
                              stream()), "maxpool2_bwd")
        torch.cuda.synchronize()
        name = f"maxpool2_bwd relu_mask={relu} add={use_add}"
        check_stores(dxm, torch.arange(dxm.n, device=DEV), name + " stores")
        g = gdy.double()
        if relu:
            g = g * (win.amax(-1) > 0)
        ref = F.one_hot(first, 4).double() * g.unsqueeze(-1)  # [N, Ho, Wo, C, 4]
        ref = ref.view(N, Ho, Wo, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(N, 2 * Ho, 2 * Wo, C)
        if use_add:
            ref = ref + ad.double()
        check(name + " (first-maximum tie rule)", dxm.body.view(N, 2 * Ho, 2 * Wo, C), ref, U_BF16 * ref.abs())


@pytest.mark.parametrize("P,C", [(1, 8), (1, 2048), (5000, 8), (5000, 2048), (1 + 2 ** 20, 8)], ids=str)
def test_colsum(P, C):
    gen = torch.Generator(device=DEV).manual_seed(P + C)
    x = rnd(P, C, gen=gen)
    X = poisoned(x, C)
    out = Guarded(C, torch.float32)
    ok(K.L.vqb_colsum(X.ptr(), out.ptr(), P, C, stream()), "colsum")
    torch.cuda.synchronize()
    check_stores(out, torch.arange(C, device=DEV), f"colsum P={P} C={C} stores")
    depth = 256 + P // 256  # fp32 adds along the longest chain (per thread, block, atomics)
    check(f"colsum P={P} C={C}", out.body, x.double().sum(0), depth * U_F32 * x.double().abs().sum(0))


@pytest.mark.parametrize("bf16", [0, 1])
def test_gauss_reparam(bf16):
    gen = torch.Generator(device=DEV).manual_seed(71)
    N, Z, S = 2, 4, 1001  # S not a multiple of any vector width
    dt = torch.bfloat16 if bf16 else torch.float32
    z = torch.randn(N, 2 * Z, S, device=DEV, generator=gen) * 2
    z[:, Z:, :5] = -10  # logvar clamped at -3
    z = z.to(dt)
    eps = torch.randn(N, Z, S, device=DEV, generator=gen).to(dt)
    Zg = Guarded(z.numel(), dt, poison="nan")
    Zg.body.copy_(z.reshape(-1))
    Eg = Guarded(eps.numel(), dt, poison="nan")
    Eg.body.copy_(eps.reshape(-1))
    out = Guarded(N * Z * S, dt)
    ok(K.L.vqb_gauss_reparam(Zg.ptr(), Eg.ptr(), out.ptr(), N, Z, S, bf16, stream()), "gauss_reparam")
    torch.cuda.synchronize()
    name = f"gauss_reparam {'bf16' if bf16 else 'fp32'} S={S}"
    check_stores(out, torch.arange(out.n, device=DEV), name + " stores")
    z64 = z.double()
    sd = torch.exp(0.5 * z64[:, Z:].clamp_min(-3)) * eps.double()
    ref = z64[:, :Z] + sd
    u = U_BF16 if bf16 else 2.0 ** -23
    check(name, out.body.view(N, Z, S), ref, u * ref.abs() + 2.0 ** -20 * sd.abs())


def test_lpips_tail_hw1():
    L = K.L
    gen = torch.Generator(device=DEV).manual_seed(81)
    N, HW, C = 3, 1, 64
    f0 = rnd(N, HW, C, gen=gen).float().relu().to(torch.bfloat16)
    f1 = rnd(N, HW, C, gen=gen).float().relu().to(torch.bfloat16)
    w = torch.rand(C, device=DEV, generator=gen) / C
    F0, F1 = poisoned(f0, C), poisoned(f1, C)
    out = Guarded(N, torch.float32)
    out.body.fill_(0.5)  # the layers accumulate into one vector
    ok(L.vqb_lpips_tail_fwd(F0.ptr(), F1.ptr(), w.data_ptr(), out.ptr(), N, HW, C, stream()), "lpips_tail_fwd")
    torch.cuda.synchronize()
    check_stores(out, torch.arange(N, device=DEV), "lpips_tail_fwd HW=1 stores")
    a = f0.double().requires_grad_(True)
    b = f1.double()

    def nrm(t):
        return t / (t.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)

    val = ((nrm(a) - nrm(b)) ** 2 * w.double()).sum(-1).mean(-1)
    check("lpips_tail_fwd HW=1", out.body, 0.5 + val.detach(), 2.0 ** -20 * (0.5 + val.detach()))
    gsc = torch.rand(N, device=DEV, generator=gen) + 0.5
    df0 = Guarded(f0.numel(), torch.bfloat16)
    ok(L.vqb_lpips_tail_bwd(F0.ptr(), F1.ptr(), w.data_ptr(), gsc.data_ptr(), df0.ptr(), N, HW, C, stream()),
       "lpips_tail_bwd")
    torch.cuda.synchronize()
    check_stores(df0, torch.arange(df0.n, device=DEV), "lpips_tail_bwd HW=1 stores")
    (gr,) = torch.autograd.grad(val, a, gsc.double())
    gr = gr * (a.detach() > 0)
    scale = gr.abs().amax(-1, keepdim=True)
    check("lpips_tail_bwd HW=1", df0.body.view(N, HW, C), gr, U_BF16 * gr.abs() + 2.0 ** -16 * scale)
