"""GPU (-m gpu): element-wise bounds of the loss and optimizer kernels of the training step against float64, in the
style and with the helpers of test_gpu_kernel_bounds.py: outputs in NaN-sentinel buffers with 4 KB guard bands (every
addressed element written, nothing else touched), inputs surrounded by NaN.

  vqb_lpips_tail_fwd / _bwd (+ _dropout)  out[n] += mean_p sum_c w_c (f0 i0 - f1 i1)^2 and d/df0 against the fp64
                                           formula (the dropout mask from vqb_lpips_dropout_mask), at every lane layout
                                           (C = 64 .. 512, VPL = 2 at C = 512), ragged and one-pixel last blocks,
                                           all-zero and tiny pixels (the |f0| == 0 branch, the 1e-10 epsilon), signed w
  vqb_lpips_dropout_mask                   bit for bit against a NumPy restatement of the documented hash
  vqb_vq_argmin                            idx equal to oracle/vq_oracle.py (ties, chunk and row tails, NaN and
                                           overflowing distances), zq = e[idx] bit for bit, sqerr within its bound
  vqb_adamw_flat / _dev                    the kernel's AdamW formula in fp64 over a grid-stride chunk range, 4 groups,
                                           skipped chunks bit for bit, the device-record path equal to the host's
  vqb_gauss_reparam_bwd                    dmean = g exactly, dlogvar within 8 u |ref|, the clamp edge at -3

Each bound is a rounding count times u = 2^-24 times the same expression on absolute values; its derivation is written
next to it. The largest max(err/bound) observed on one H100 80GB HBM3 (700 W power limit) is noted beside each. Mutation
checks prove that the bounds bite.

`python -m pytest -m gpu -q tests/test_gpu_loss_optim_bounds.py -s` prints one max(err/bound) line per case.
"""
import ctypes
import math
import types

import numpy as np
import pytest
import torch

from test_gpu_kernel_bounds import (DEV, GUARD_BYTES, U_BF16, U_F32, Guarded, K, check, check_bits,  # noqa: F401
                                    check_stores, lib, ok, poisoned, rejects, rnd, stream)

pytestmark = pytest.mark.gpu

u = U_F32


def nan_guarded(vals):
    """A flat copy of `vals` with NaN on both sides."""
    G = Guarded(vals.numel(), vals.dtype, poison="nan")
    G.body.copy_(vals.reshape(-1))
    return G


class GuardedBytes:
    """uint8 [guard | body | guard] with a fill byte the kernels never write (the guards) or a chosen one (inputs)."""

    def __init__(self, n, fill=0xA5):
        self.n, self.g = int(n), GUARD_BYTES
        self.buf = torch.full((self.n + 2 * self.g,), fill, dtype=torch.uint8, device=DEV)

    @property
    def body(self):
        return self.buf[self.g:self.g + self.n]

    def ptr(self):
        return self.buf.data_ptr() + self.g


# ---------------------------------------------------------------------------------------------------- LPIPS tail
LP_EPS = float(torch.tensor(1e-10, dtype=torch.float32))  # the kernels add 1e-10f, not the double 1e-10


def lpips_geometry(HW, C):
    """The launch of lpips_tail_*_impl: G lanes per pixel, VPL vectors per lane, pixels per block, blocks per image and
    pixel passes per warp."""
    V = C // 8
    G = min(32, V)
    VPL, ppw = V // G, 32 // G
    ppb = max(-(-HW // 528), 2 * 8 * ppw)
    return G, VPL, ppb, -(-HW // ppb), -(-ppb // (8 * ppw))


def lpips_roundings(HW, C):
    """(n_fwd, n_bwd): rounding counts of the longest fp32 chains (first order, a rounding <= u of its value)."""
    G, VPL, _, nblk, passes = lpips_geometry(HW, C)
    lg = int(math.log2(G))
    n_s = 8 * VPL + lg        # |f|^2: 8 VPL fused multiply-adds per lane, log2 G shuffle adds (positive terms)
    k_inv = n_s / 2 + 3       # i = 1 / (sqrt(s) + eps): sqrt halves s's relative error (+1), + eps (+1), 1 / x (+1)
    k_t = k_inv + 2           # t = f0 i0 - f1 i1: a product, the difference (+2): |dt| <= k_t u (|f0| i0 + |f1| i1)
    # forward: w t^2 (t^2 doubles t's coefficient, +1; w * +1), then the sums: the lane's 8 VPL channels, its pixel
    # passes, the warp and block trees (5 + 5), inv_hw and the product (2), the atomicAdd chain over the image's blocks
    # onto the pre-filled out (nblk)
    n_fwd = 2 * k_t + 2 + 8 * VPL + passes + 10 + 2 + nblk
    # backward: q = 2 w t (2 w exact, * t +1); dot = sum q f0 (+1 per product, the lane's 8 VPL, log2 G shuffle adds);
    # k2 = dot i0 i0 / |f0| (two i0, |f0| = sqrt(s0) with n_s / 2 + 1, three roundings); q i0 or k2 f0 (+1), their
    # difference (+1), gn = g * inv_hw (2) and gn * (+1); the bf16 rounding's (1 + 2^-8) factor on the fp32 error (+1)
    k_q = k_t + 1
    k_k2 = (k_q + 1 + 8 * VPL + lg) + 2 * k_inv + (n_s / 2 + 1) + 3
    n_bwd = max(k_q + k_inv, k_k2) + 1 + 1 + 3 + 1
    return n_fwd, n_bwd


def lpips_ref(f0, f1, w_eff, out0, g):
    """fp64 forward value, its absolute-value sum S, backward d/df0 (gated by f0 > 0) and its sensitivity on |q| i0 and
    |k2| |f0|. w_eff broadcasts against [N, HW, C] (w, or w * 2 * mask for the dropout variants)."""
    a, b = f0.double(), f1.double()
    HW = a.shape[1]
    na = a.square().sum(-1, keepdim=True).sqrt()
    nb = b.square().sum(-1, keepdim=True).sqrt()
    i0, i1 = 1.0 / (na + LP_EPS), 1.0 / (nb + LP_EPS)
    t = a * i0 - b * i1
    A = a.abs() * i0 + b.abs() * i1
    per_pix = (w_eff * t * t).sum(-1)
    val = out0.double() + per_pix.sum(-1) / HW
    S = out0.double().abs() + (w_eff.abs() * A * A).sum(-1).sum(-1) / HW
    q, Q = 2 * w_eff * t, 2 * w_eff.abs() * A
    live = na > 0
    k2 = torch.where(live, (q * a).sum(-1, keepdim=True) * i0 * i0 / na, 0.0)
    K2 = torch.where(live, (Q * a.abs()).sum(-1, keepdim=True) * i0 * i0 / na, 0.0)
    gn = (g.double() / HW).view(-1, 1, 1)
    gate = a > 0
    d = gn * (q * i0 - k2 * a) * gate
    sens = gn.abs() * (Q * i0 + K2 * a.abs()) * gate
    return types.SimpleNamespace(val=val, S=S, per_pix=per_pix, d=d, sens=sens, t=t, q=q, i0=i0, k2=k2, gn=gn,
                                 gate=gate)


def lpips_inputs(N, HW, C, seed, signed_w):
    """Post-ReLU feature pairs of a reconstruction and its target (f1 = f0's pre-activation + noise: t cancels), with an
    all-zero f0 pixel, an all-zero f1 pixel and a tiny f0 pixel (|f0| ~ 1e-8, where the 1e-10 epsilon shows)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    pre = torch.randn(N, HW, C, device=DEV, generator=gen)
    f0 = pre.relu()
    f1 = (pre + 0.3 * torch.randn(N, HW, C, device=DEV, generator=gen)).relu()
    f0[0, 0] = 0
    f1[1 % N, HW - 1] = 0
    f0[2 % N, HW // 2] *= 2.0 ** -30
    if signed_w:
        w = torch.randn(C, device=DEV, generator=gen) / C
    else:
        w = torch.rand(C, device=DEV, generator=gen) * (2.0 / C)
    g = torch.rand(N, device=DEV, generator=gen) + 0.5
    return f0.to(torch.bfloat16), f1.to(torch.bfloat16), w, g


# (C, HW): every lane layout (G = 8, 16, 32 lanes per pixel; VPL = 2 at C = 512), 65536 pixels (many blocks adding
# into out[n]), ragged pixel passes and blocks, fewer pixels than one warp pass (HW = 3) or one pixel, and HW = 1025 at
# C = 64: 16 blocks of 64 pixels and a last block of one pixel.
LPIPS_CASES = [(64, 65536), (64, 1369), (64, 3), (64, 1025), (128, 1000), (256, 97), (512, 64), (512, 1)]
# Observed max(err/bound) on the H100 noted above: forward 0.028; backward 0.995, all of it the bf16 rounding (the share
# of the n_bwd u term, printed as the accumulation share, is 0.021).


@pytest.mark.parametrize("C,HW", LPIPS_CASES, ids=lambda v: str(v))
def test_lpips_tail_bounds(C, HW):
    L = K.L
    N = 3
    signed = (C, HW) == (256, 97)
    f0, f1, w, g = lpips_inputs(N, HW, C, seed=C * 7919 + HW, signed_w=signed)
    F0, F1, Wg, Gg = poisoned(f0, C), poisoned(f1, C), nan_guarded(w), nan_guarded(g)
    out0 = torch.tensor([0.25e-2, -0.5e-2, 1e-2], device=DEV)
    seed = (0x9E3779B97F4A7C15 * (C + HW)) % 2 ** 64
    n_fwd, n_bwd = lpips_roundings(HW, C)
    _, _, ppb, nblk, _ = lpips_geometry(HW, C)
    if HW == 1025:
        assert HW - (nblk - 1) * ppb == 1  # the case's reason to exist: a one-pixel last block

    def fwd(drop):
        out = Guarded(N, torch.float32)
        out.body.copy_(out0)  # the five LPIPS layers accumulate into one vector: out is added to
        if drop:
            rc = L.vqb_lpips_tail_fwd_dropout(F0.ptr(), F1.ptr(), Wg.ptr(), out.ptr(), N, HW, C, seed, stream())
        else:
            rc = L.vqb_lpips_tail_fwd(F0.ptr(), F1.ptr(), Wg.ptr(), out.ptr(), N, HW, C, stream())
        ok(rc, "lpips_tail_fwd")
        torch.cuda.synchronize()
        check_stores(out, torch.arange(N, device=DEV), f"lpips fwd C={C} HW={HW} stores")
        return out

    def bwd(drop):
        df0 = Guarded(N * HW * C, torch.bfloat16)
        if drop:
            rc = L.vqb_lpips_tail_bwd_dropout(F0.ptr(), F1.ptr(), Wg.ptr(), Gg.ptr(), df0.ptr(), N, HW, C, seed,
                                              stream())
        else:
            rc = L.vqb_lpips_tail_bwd(F0.ptr(), F1.ptr(), Wg.ptr(), Gg.ptr(), df0.ptr(), N, HW, C, stream())
        ok(rc, "lpips_tail_bwd")
        torch.cuda.synchronize()
        check_stores(df0, torch.arange(df0.n, device=DEV), f"lpips bwd C={C} HW={HW} stores")
        return df0

    mask = GuardedBytes(N * HW * C)
    ok(L.vqb_lpips_dropout_mask(seed, N, HW, C, mask.ptr(), stream()), "lpips_dropout_mask")
    torch.cuda.synchronize()
    keep = mask.body.view(N, HW, C).double()
    for drop in (False, True):
        tag = f"lpips{' dropout' if drop else ''} C={C} HW={HW}{' signed w' if signed else ''}"
        w_eff = w.double() * 2 * keep if drop else w.double()
        r = lpips_ref(f0, f1, w_eff, out0, g)
        out = fwd(drop)
        # forward: |got - val| <= n_fwd u S, S = the same sums on |w| (|f0| i0 + |f1| i1)^2 and |out0|
        check(tag + " fwd", out.body, r.val, n_fwd * u * r.S)
        # backward, rounded to bf16: 2^-8 |ref| + n_bwd u gn (|q| i0 + |k2| |f0|) on the absolute-value terms
        df0 = bwd(drop)
        got = df0.body.view(N, HW, C)
        bound = U_BF16 * r.d.abs() + n_bwd * u * r.sens
        check(tag + " bwd", got, r.d, bound, acc=(U_BF16 * r.d.abs(), n_bwd * u * r.sens))
        check_bits(tag + " bwd", df0.bits(), bwd(drop).bits())

        if HW == 1025 and not drop:  # the forward bound bites: the reference without the one-pixel last block
            rejects(tag + " fwd: reference without the last pixel", out.body, r.val - r.per_pix[:, -1] / HW,
                    n_fwd * u * r.S)
        if C == 512 and HW == 64 and not drop:  # the backward bound bites: k2 dropped at the pixel where it weighs most
            n, p = divmod(int((r.gn * r.k2 * f0.double() * r.gate).abs().amax(-1).argmax()), HW)
            d_mut = r.d.clone()
            d_mut[n, p] = (r.gn * r.q * r.i0 * r.gate)[n, p]
            rejects(tag + f" bwd: reference without the k2 term at pixel ({n}, {p})", got, d_mut, bound)
        if C == 512 and HW == 64 and drop:
            # the mask of one 8-channel vector in the second-vector slot (vectors 32..63 of a lane) taken from the next
            # vector, at the (pixel, vector) where that changes the value most among channels with f0 > 0 (elsewhere
            # the gradient is gated to 0 whatever the mask)
            kv, tv, gv = keep.view(N, HW, 64, 8), r.t.view(N, HW, 64, 8), r.gate.view(N, HW, 64, 8)
            delta = (w.double().view(64, 8)[32:63] * 2 * (kv[:, :, 33:64] - kv[:, :, 32:63]) * tv[:, :, 32:63] ** 2
                     * gv[:, :, 32:63])
            n, p, j = (int(x) for x in np.unravel_index(int(delta.sum(-1).abs().argmax()), (N, HW, 31)))
            j += 32
            km = keep.clone().view(N, HW, 64, 8)
            km[n, p, j] = km[n, p, j + 1]
            rm = lpips_ref(f0, f1, w.double() * 2 * km.view(N, HW, C), out0, g)
            what = f" mask of vector {j} at pixel ({n}, {p}) shifted by one vector"
            rejects(tag + " fwd:" + what, out.body, rm.val, n_fwd * u * r.S)
            rejects(tag + " bwd:" + what, got, rm.d, bound)


def dropout_mask_np(seed, N, HW, C):
    """The documented keep bits: element e = (n HW + p) C + c is bit e % 32 of the upper 32 bits of the splitmix64
    finaliser of seed + (e / 32 + 1) * 0x9E3779B97F4A7C15 (uint64 arithmetic, wrapping)."""
    e = np.arange(N * HW * C, dtype=np.uint64)
    z = np.uint64(seed) + ((e >> np.uint64(5)) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z ^= z >> np.uint64(31)
    return (((z >> np.uint64(32)) >> (e & np.uint64(31))) & np.uint64(1)).astype(np.uint8).reshape(N, HW, C)


@pytest.mark.parametrize("seed", [0, 1, 2 ** 64 - 1])
@pytest.mark.parametrize("N,HW,C", [(3, 5, 8), (3, 37, 72)])  # N HW C = 120, 7992: not multiples of 32
def test_lpips_dropout_mask_bits(seed, N, HW, C):
    mask = GuardedBytes(N * HW * C)
    ok(K.L.vqb_lpips_dropout_mask(seed, N, HW, C, mask.ptr(), stream()), "lpips_dropout_mask")
    torch.cuda.synchronize()
    b = mask.buf.cpu().numpy()
    assert (b[:mask.g] == 0xA5).all() and (b[mask.g + mask.n:] == 0xA5).all(), "mask written outside [N][HW][C]"
    got = b[mask.g:mask.g + mask.n].reshape(N, HW, C)
    want = dropout_mask_np(seed, N, HW, C)
    print(f"  dropout mask seed={seed} N={N} HW={HW} C={C}: mismatches {(got != want).sum()}, keep "
          f"{want.mean():.3f}", flush=True)
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------- VQ search
def vq_oracle(z, e):
    from oracle import vq_oracle as VQ

    with np.errstate(over="ignore", invalid="ignore"):
        return VQ.vq_argmin(z, e)


def vq_run(z, e, sq0=None):
    """-> (idx, zq, sqerr or None). idx (int64) lives in a float32 sentinel buffer of 2M words: an index < 2^31 writes
    two words that are no NaN payload, so check_stores sees every write."""
    M, D = z.shape
    Zg, Eg = nan_guarded(torch.from_numpy(z).to(DEV)), nan_guarded(torch.from_numpy(e).to(DEV))
    I = Guarded(2 * M, torch.float32)
    Q = Guarded(M * D, torch.float32)
    S = None
    if sq0 is not None:
        S = Guarded(1, torch.float32)
        S.body.fill_(sq0)
    ok(K.L.vqb_vq_argmin(Zg.ptr(), Eg.ptr(), I.ptr(), Q.ptr(), S.ptr() if S else None, M, e.shape[0], D, stream()),
       "vq_argmin")
    torch.cuda.synchronize()
    check_stores(I, torch.arange(2 * M, device=DEV), f"vq idx M={M} stores")
    check_stores(Q, torch.arange(M * D, device=DEV), f"vq zq M={M} D={D} stores")
    if S is not None:
        check_stores(S, torch.arange(1, device=DEV), "vq sqerr stores")
    return I.body.view(torch.int64).cpu().numpy(), Q.body.view(M, D).cpu().numpy(), S


def vq_data(M, ncode, D, seed):
    rng = np.random.default_rng(seed)
    if D <= 3:  # coarse grids: exact distance ties between codes of different lanes and chunks; the first index wins
        e = (rng.integers(-4, 5, size=(ncode, D)) / 4).astype(np.float32)
        z = (rng.integers(-8, 9, size=(M, D)) / 8).astype(np.float32)
    else:
        e = rng.standard_normal((ncode, D)).astype(np.float32)
        z = rng.standard_normal((M, D)).astype(np.float32)
        if ncode > 4:
            e[ncode // 2] = e[3]  # a duplicate code in another lane (and, for ncode > chunk, another chunk): 3 wins
            z[9] = e[3]
        z[8] = e[ncode - 1]  # an exact hit on the last code (the one-code last chunk at ncode = 1025)
    return z, e


# D = 256 stages codes in chunks of 64, D = 255 in chunks of 128, D <= 64 in chunks of 1024: ncode = 1025 leaves a
# one-code last chunk, ncode = 300 at D = 256 five chunks, the last of 44. M = 20000 rows exceed the grid of 2 x 132
# blocks x 32 rows, so the row grid-stride loop runs (at ncode <= 33, where the NumPy oracle stays cheap).
VQ_CASES = [(D, ncode, 20000 if ncode <= 33 else 257) for D in (1, 3, 16, 17, 64, 255, 256) for ncode in (1, 33, 1025)]
VQ_CASES += [(256, 300, 2000)]
# Observed max(err/bound) of sqerr on the H100 noted above: 0.033 (the atomic order varies from run to run).


@pytest.mark.parametrize("D,ncode,M", VQ_CASES, ids=lambda v: str(v))
def test_vq_argmin_bounds(D, ncode, M):
    z, e = vq_data(M, ncode, D, seed=D * 1000 + ncode)
    want = vq_oracle(z, e)
    sq0 = 0.75
    idx, zq, S = vq_run(z, e, sq0)
    name = f"vq D={D} K={ncode} M={M}"
    bad = int((idx != want).sum())
    print(f"  {name}: index mismatches {bad}", flush=True)
    assert bad == 0, f"{name}: first mismatch at row {int(np.argmax(idx != want))}"
    assert np.array_equal(zq.view(np.int32), e[want].view(np.int32)), f"{name}: zq is not e[idx] bit for bit"
    # sqerr: per row (zq - z) and its square or fma (2 + 1 roundings, the first term), the lane's ceil(D/32) terms, the
    # 5-level shuffle tree, then the atomicAdd chain of M rows onto the pre-filled value: M + ceil(D/32) + 7 roundings
    # of positive terms (<= D + M + 6 for D >= 2)
    ref = sq0 + float(((e[want].astype(np.float64) - z) ** 2).sum())
    nr = M + -(-D // 32) + 7
    check(name + " sqerr", S.body, torch.tensor([ref], device=DEV, dtype=torch.float64), nr * u * ref)
    idx2, zq2, _ = vq_run(z, e, None)  # sqerr = NULL
    assert np.array_equal(idx2, want) and np.array_equal(zq2.view(np.int32), zq.view(np.int32)), name + " sqerr=NULL"


@pytest.mark.parametrize("D,ncode", [(16, 1025), (256, 300)], ids=str)
def test_vq_argmin_non_finite(D, ncode):
    """np.argmin's rule: the first NaN distance wins, an all-+inf row gets 0; the index stays in [0, K)."""
    M = 300
    rng = np.random.default_rng(D + ncode)
    e = rng.standard_normal((ncode, D)).astype(np.float32)
    z = rng.standard_normal((M, D)).astype(np.float32)
    z[3, D // 2] = np.nan      # every distance of row 3 is NaN: index 0
    z[10] = 1e30               # |z - e|^2 overflows for every code: all +inf, index 0
    z[20, 0] = 1.5e19          # codes 0..2 overflow (9e38), the others stay finite (~2.25e38, ties): a finite one wins
    e[0:3, 0] = -1.5e19
    want = vq_oracle(z, e)
    assert want[3] == 0 and want[10] == 0 and want[20] >= 3
    idx, zq, _ = vq_run(z, e)
    print(f"  vq non-finite z D={D} K={ncode}: index mismatches {(idx != want).sum()}, rows 3/10/20 -> "
          f"{idx[3]}/{idx[10]}/{idx[20]}", flush=True)
    assert np.array_equal(idx, want)
    assert np.array_equal(zq.view(np.int32), e[want].view(np.int32))

    e[5, 7 % D] = np.nan       # a NaN code: its distance is NaN for every row, so it wins everywhere but row 3
    want = vq_oracle(z, e)
    assert want[3] == 0 and (np.delete(want, 3) == 5).all()
    idx, zq, _ = vq_run(z, e)
    print(f"  vq NaN code D={D} K={ncode}: index mismatches {(idx != want).sum()}", flush=True)
    assert np.array_equal(idx, want)
    assert np.array_equal(zq.view(np.int32), e[want].view(np.int32))


# ---------------------------------------------------------------------------------------------------- AdamW
ADAMW_GROUPS = (  # lr, beta1, beta2, eps, weight_decay; betas >= 0.5, so 1 - beta is exact in fp32 (Sterbenz)
    (1e-3, 0.9, 0.95, 1e-8, 1e-3),        # the trainers' setting
    (3e-4, 0.8, 0.999, 1e-6, 0.1),
    (2e-2, 0.9999, 0.99999, 1e-5, 0.0),   # slow betas: the bias corrections still move at step 10^4
    (5e-3, 0.5, 0.9, 1e-3, 0.01),
)
NCHUNK = 3001  # > 16 x 132 blocks: the chunk grid-stride loop runs
GRAD_SCALE = 0.37
# Observed max(err/bound) on the H100 noted above: p 0.571, m 0.623, v 0.694.


def adamw_groups(step):
    import native

    arr = (native.VqbAdamwGroup * 4)()
    for i, (lr, b1, b2, eps, wd) in enumerate(ADAMW_GROUPS):
        arr[i].lr, arr[i].beta1, arr[i].beta2, arr[i].eps, arr[i].weight_decay, arr[i].step = lr, b1, b2, eps, wd, step
    return arr


def adamw_ref(p, g, m, v, cg, rec, gs):
    """The kernel's formula in fp64 on the fp32 values: p (1 - lr wd) - (lr / bc1) m' / (sqrt(v') / bc2s + eps),
    m' = m + (1 - b1)(g gs - m), v' = b2 v + (1 - b2)(g gs)^2; chunks of group 255 unchanged. rec [7, 4] fp64 holds the
    record's lr, beta1, beta2, eps, wd, bc1, bc2_sqrt. -> (p', m', v') and their bounds."""
    grp = cg.long().repeat_interleave(1024)
    act = grp < 4
    lr, b1, b2, eps, wd, bc1, bc2s = (rec[k][grp.clamp_max(3)] for k in range(7))
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    gr = g * gs
    m1 = m + (1 - b1) * (gr - m)
    v1 = b2 * v + (1 - b2) * gr * gr
    den = v1.sqrt() / bc2s + eps
    step = lr / bc1
    p1 = p * (1 - lr * wd) - step * m1 / den
    # m': g * gs, gr - m, (1 - b1) * and + (or one fma): 4 roundings of Sm = |m| + (1 - b1)(|gr| + |m|)
    Sm = m.abs() + (1 - b1) * (gr.abs() + m.abs())
    bm = 4 * u * Sm
    # v': gr (twice, +2), (1 - b2) * gr (+1), * gr (+1), the sum (+1) over positive terms: 5 u v'
    bv = 5 * u * v1
    # p': lr wd, 1 - x, p * decay (3 u |p|); den = sqrt(v') / bc2s + eps: 5 u / 2 + 1 + 1 + 1 relative; m' / den: 4 u Sm
    # + (5.5 + 1) u |m'| <= 10.5 u Sm (over den); lr / bc1 and step * (+2): 12.5 u step Sm / den; the final difference
    # u |p'| <= u (|p| + step Sm / den): 4 u |p| + 13.5 u step Sm / den
    bp = 4 * u * p.abs() + 13.5 * u * step * Sm / den
    keep = ~act
    p1, m1, v1 = torch.where(keep, p, p1), torch.where(keep, m, m1), torch.where(keep, v, v1)
    zero = torch.zeros_like(bp)
    return (p1, m1, v1), (torch.where(keep, zero, bp), torch.where(keep, zero, bm), torch.where(keep, zero, bv))


@pytest.mark.parametrize("step", [1, 10000])
def test_adamw_flat_bounds(step):
    L = K.L
    n = NCHUNK * 1024
    gen = torch.Generator(device=DEV).manual_seed(step)
    p0 = torch.randn(n, device=DEV, generator=gen)
    g0 = torch.randn(n, device=DEV, generator=gen) * 10 ** (torch.rand(n, device=DEV, generator=gen) * 4 - 3)
    m0 = torch.randn(n, device=DEV, generator=gen) * 0.01
    v0 = torch.rand(n, device=DEV, generator=gen) * 1e-3
    cg = torch.randint(0, 5, (NCHUNK,), device=DEV, generator=gen).to(torch.uint8)
    cg[cg == 4] = 255  # interleaved chunks without a gradient
    assert all(int((cg == k).sum()) > 100 for k in (0, 1, 2, 3, 255))
    CG = GuardedBytes(NCHUNK, fill=0)  # group 0 around the table: an over-read would update the guard bands of p, m, v
    CG.body.copy_(cg)
    Gg = nan_guarded(g0)
    groups = adamw_groups(step)
    rec_host = (ctypes.c_float * 28)()
    ok(L.vqb_adamw_fill_record(4, groups, rec_host), "adamw_fill_record")
    rec32 = torch.tensor(list(rec_host), dtype=torch.float32, device=DEV)
    REC = nan_guarded(rec32)

    def run(dev):
        P, M, V = (Guarded(n, torch.float32) for _ in range(3))
        for B, x in ((P, p0), (M, m0), (V, v0)):
            B.body.copy_(x)
        if dev:
            rc = L.vqb_adamw_flat_dev(P.ptr(), Gg.ptr(), M.ptr(), V.ptr(), CG.ptr(), NCHUNK, REC.ptr(), GRAD_SCALE,
                                      stream())
        else:
            rc = L.vqb_adamw_flat(P.ptr(), Gg.ptr(), M.ptr(), V.ptr(), CG.ptr(), NCHUNK, 4, groups, GRAD_SCALE,
                                  stream())
        ok(rc, "adamw_flat" + ("_dev" if dev else ""))
        torch.cuda.synchronize()
        for B, nm in ((P, "p"), (M, "m"), (V, "v")):
            check_stores(B, torch.arange(n, device=DEV), f"adamw {nm} stores")
        return P, M, V

    P, M, V = run(False)
    name = f"adamw step={step} chunks={NCHUNK}"
    gs = float(np.float32(GRAD_SCALE))
    rec = rec32.double().view(7, 4)
    (pr, mr, vr), (bp, bm, bv) = adamw_ref(p0, g0, m0, v0, cg, rec, gs)
    check(name + " p", P.body, pr, bp)
    check(name + " m", M.body, mr, bm)
    check(name + " v", V.body, vr, bv)
    skip = (cg == 255).repeat_interleave(1024)
    for B, x, nm in ((P, p0, "p"), (M, m0, "m"), (V, v0, "v")):
        assert torch.equal(B.body.view(torch.int32)[skip], x.view(torch.int32)[skip]), f"{name}: skipped {nm} changed"
    again = run(False)
    check_bits(name, torch.cat([B.bits() for B in (P, M, V)]), torch.cat([B.bits() for B in again]))
    devrun = run(True)
    same = all(torch.equal(a.bits(), b.bits()) for a, b in zip((P, M, V), devrun))
    print(f"  {name}: device-record path bit-identical={same}", flush=True)
    assert same, f"{name}: vqb_adamw_flat_dev differs from vqb_adamw_flat on the same record"

    # the bounds bite
    got = torch.cat([P.body, M.body, V.body])
    bound = torch.cat([bp, bm, bv])
    b1, b2 = rec[1].clone(), rec[2].clone()
    rec_t1 = rec.clone()
    rec_t1[5] = 1 - b1 ** (step + 1)
    rec_t1[6] = (1 - b2 ** (step + 1)).sqrt()
    rejects(name + ": bias correction of step t+1", got, torch.cat(adamw_ref(p0, g0, m0, v0, cg, rec_t1, gs)[0]), bound)
    rejects(name + ": without grad_scale", got, torch.cat(adamw_ref(p0, g0, m0, v0, cg, rec, 1.0)[0]), bound)
    c = int((cg == 0).nonzero()[0])
    cg_mut = cg.clone()
    cg_mut[c] = 1
    rejects(name + f": chunk {c} taken as group 1", got, torch.cat(adamw_ref(p0, g0, m0, v0, cg_mut, rec, gs)[0]),
            bound)


# ---------------------------------------------------------------------------------------------------- reparam gradient
def test_gauss_reparam_bwd_bounds():
    L = K.L
    N, Z, S = 2, 3, 1001  # S ragged against every vector width
    gen = torch.Generator(device=DEV).manual_seed(91)
    z = torch.randn(N, 2 * Z, S, device=DEV, generator=gen)
    z[:, Z:] *= 4  # logvar over both sides of the clamp at -3
    lo = torch.nextafter(torch.tensor(-3.0), torch.tensor(-math.inf)).item()
    z[:, Z:, 0] = -3.0  # the clamp passes the gradient at exactly -3
    z[:, Z:, 1] = lo    # and blocks it one fp32 step below
    z[:, Z:, 2] = 80.0  # exp(40): large, finite
    g = torch.randn(N, Z, S, device=DEV, generator=gen)
    eps = torch.randn(N, Z, S, device=DEV, generator=gen)
    Zg, Gg, Eg = nan_guarded(z), nan_guarded(g), nan_guarded(eps)
    dz = Guarded(N * 2 * Z * S, torch.float32)
    ok(L.vqb_gauss_reparam_bwd(Gg.ptr(), Zg.ptr(), Eg.ptr(), dz.ptr(), N, Z, S, stream()), "gauss_reparam_bwd")
    torch.cuda.synchronize()
    name = f"gauss_reparam_bwd N={N} Z={Z} S={S}"
    check_stores(dz, torch.arange(dz.n, device=DEV), name + " stores")
    d = dz.body.view(N, 2 * Z, S)
    assert torch.equal(d[:, :Z].contiguous().view(torch.int32), g.view(torch.int32)), name + ": dmean is not g"
    lv = z[:, Z:].double()
    ref = torch.where(lv >= -3, g.double() * eps.double() * 0.5 * torch.exp(0.5 * lv), 0.0)
    # expf (no fast math) is within 2 ulp <= 4 u relative; g * eps, * exp, * 0.5 (exact): 3 roundings -> 7 u; 8 u with
    # the first-order slack of composing them. Observed max(err/bound) on the H100 noted above: 0.36.
    check(name + " dlogvar", d[:, Z:], ref, 8 * u * ref.abs())
    assert (d[:, Z:, 0] != 0).all(), "the gradient must pass at logvar = -3"
    assert (d[:, Z:, 1] == 0).all(), "the gradient must be 0 below -3"
    assert torch.isfinite(d[:, Z:, 2]).all() and (d[:, Z:, 2] != 0).all()
