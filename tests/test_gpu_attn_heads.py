"""GPU (-m gpu): the attention forward and backward (vqb_attn_fwd_hd / vqb_attn_bwd_hd) at every head size tae.AttnBlock
can produce, 8 to 112 channels in steps of 8.

Kernel level, with the bounds and guarded buffers of test_gpu_kernel_bounds.py: out and lse within the element-wise
forward bound of a float64 reference, dq / dk / dv per (n, head, token) row within 2^-6 of the row's fp64 norm plus the
error the flash backward inherits; NaN-poisoned inputs and sentinel-filled outputs with 4 KB guard bands (every
addressed element written, nothing else); reruns bit-identical. Heads of 8 * odd channels (8, 24, ..., 104) run Q.K^T
over a zero-filled padding column block, and heads above 64 split the dK / dV work across two CTAs per key tile.

Against SDPA at the 8 x 6144-token mid-block shape, with the rule of test_gpu_tae.py / test_gpu_tae_train.py: ours
within 1.5 x the bf16 SDPA peer's relative L2 error to the fp32 SDPA truth (TF32 off) plus 2e-3, for the forward and
for each of dq, dk, dv.
"""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_kernel_bounds import (DEV, U_BF16, Guarded, K, attn_bwd_inherent, attn_check_fwd, attn_inputs,
                                    attn_run_fwd, check, check_bits, check_stores, lib, ok, rnd, rowwise,
                                    stream)  # noqa: F401  (lib: the module fixture that loads the library)
from test_gpu_tae import check as check_fwd_sdpa
from test_gpu_tae import tf32_off
from test_gpu_tae_train import check as check_bwd_sdpa

pytestmark = pytest.mark.gpu

HEAD_DIMS = list(range(8, 113, 8))
CASES = [
    # T, heads, N, q scale, max key in the ragged tail, q = 0
    (1, 1, 1, 0.5, False, False),
    (65, 3, 3, 3.0, True, False),
    (65, 3, 1, 1.0, False, True),
    (129, 8, 1, 0.5, True, False),
    (1000, 1, 3, 3.0, True, False),
    (4097, 1, 1, 0.5, True, False),
]


def _bwd(Q, out, DO, lse, N, T, C, hd):
    heads = C // hd
    dvec = Guarded(N * heads * T, torch.float32)
    dq = Guarded(N * T * 3 * C, torch.bfloat16)
    ok(K.L.vqb_attn_bwd_hd(Q.ptr(), out.ptr(), DO.ptr(), lse.ptr(), dvec.ptr(), dq.ptr(), N, T, C, hd, stream()),
       "attn_bwd_hd")
    torch.cuda.synchronize()
    return dvec, dq


@pytest.mark.parametrize("hd", HEAD_DIMS)
@pytest.mark.parametrize("T,heads,N,qs,tail,qzero", CASES, ids=lambda v: str(v))
def test_attention_head_bounds(hd, T, heads, N, qs, tail, qzero):
    scale = hd ** -0.5
    qkv, C = attn_inputs(T, heads, N, qs, tail, qzero, hd, seed=1000 * hd + T + heads)
    Q = Guarded(qkv.numel(), torch.bfloat16, poison="nan")
    Q.body.copy_(qkv.reshape(-1))
    out = Guarded(N * T * C, torch.bfloat16)
    lse = Guarded(N * heads * T, torch.float32)
    ok(K.L.vqb_attn_fwd_hd(Q.ptr(), out.ptr(), lse.ptr(), N, T, C, hd, stream()), "attn_fwd_hd")
    torch.cuda.synchronize()
    name = f"attn hd={hd} T={T} heads={heads} N={N} qscale={qs}{' tail-max' if tail else ''}{' q=0' if qzero else ''}"
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
    gen = torch.Generator(device=DEV).manual_seed(T + hd)
    dout = rnd(N, T, C, gen=gen)
    DO = Guarded(dout.numel(), torch.bfloat16, poison="nan")
    DO.body.copy_(dout.reshape(-1))
    dvec, dq = _bwd(Q, out, DO, lse, N, T, C, hd)
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
    _, dq2 = _bwd(Q, out, DO, lse, N, T, C, hd)
    check_bits(name + " bwd", dq.bits(), dq2.bits())


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_attention_heads_match_sdpa_forward_and_backward(hd):
    """ops.attention_hd_train at the 48 x 256^2 mid-block shape (8 heads x 6144 tokens, batch 2)."""
    import ops

    g = torch.Generator(device="cuda").manual_seed(hd + 17)
    N, T, heads = 2, 6144, 8
    C = heads * hd
    qkv = torch.randn(N, 6, 32, 32, 3 * C, device="cuda", generator=g).bfloat16()
    dout = torch.randn(N, 6, 32, 32, C, device="cuda", generator=g).bfloat16()
    q0 = qkv.clone().requires_grad_(True)
    out = ops.attention_hd_train(q0, heads, hd)
    out.backward(dout)

    def sdpa(u, d):
        u = u.detach().clone().requires_grad_(True)
        q, k, v = (a.reshape(N, T, heads, hd).permute(0, 2, 1, 3) for a in u.reshape(N, T, 3 * C).chunk(3, -1))
        o = F.scaled_dot_product_attention(q, k, v)
        o.permute(0, 2, 1, 3).reshape(u.shape[:-1] + (C,)).backward(d.to(u.dtype))
        return o.detach(), u.grad

    with tf32_off():
        to, tg = sdpa(qkv.float(), dout)
    po, pg = sdpa(qkv, dout)
    ours = out.detach().reshape(N, T, heads, hd).permute(0, 2, 1, 3)
    check_fwd_sdpa(f"attention heads of {hd}", ours, to, po, torch.bfloat16)
    for i, part in enumerate("qkv"):
        sl = slice(i * C, (i + 1) * C)
        check_bwd_sdpa(f"attention heads of {hd} d{part}", q0.grad[..., sl], tg[..., sl], pg[..., sl])
