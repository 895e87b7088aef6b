#!/usr/bin/env python
"""Attention-core benchmark: vqb_attn_fwd_hd and vqb_attn_bwd_hd against F.scaled_dot_product_attention in bf16, per head
size, at tae.AttnBlock's mid-block shape.

    python tools/attn_bench.py                      # every supported head size, 8 heads x 6144 tokens, batch 1
    python tools/attn_bench.py --hd 16 112 --tokens 6144 --steps 50

6144 tokens is the mid block of a 48x256^2 clip (6 x 32 x 32 latent voxels). Ours runs on the same [N, T, 3C] qkv
layout the module feeds it; SDPA takes q, k, v as [N, heads, T, head_dim] views of that tensor (the rearrange tae.py
does), so its time includes no copy. The backward time of each is the backward alone (vqb_attn_bwd_hd: the D = rowsum
kernel, dK/dV and dQ; SDPA: its autograd backward given a saved forward). CUDA events around --steps calls after
--warmup calls. One JSON line per head size with ms per call, TFLOP/s of the attention matmuls (forward 4 T^2 d per
head, backward 10 T^2 d: the algorithm's, not counting recomputation), our time over SDPA's, and the card's name and
power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
sys.path.insert(1, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from infer_bench import card  # noqa: E402


def event_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    import native
    import ops

    ap = argparse.ArgumentParser()
    ap.add_argument("--hd", type=int, nargs="*", default=list(ops.ATTN_HEAD_DIMS))
    ap.add_argument("--tokens", type=int, default=6144)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attn_bench: needs a CUDA device")
    L = native.load()
    info = card()
    N, T, heads = a.batch, a.tokens, a.heads
    for hd in a.hd:
        C = heads * hd
        g = torch.Generator(device="cuda").manual_seed(hd)
        qkv = torch.randn(N, T, 3 * C, device="cuda", generator=g).bfloat16()
        dout = torch.randn(N, T, C, device="cuda", generator=g).bfloat16()
        out = torch.empty(N, T, C, device="cuda", dtype=torch.bfloat16)
        lse = torch.empty(N, heads, T, device="cuda", dtype=torch.float32)
        dvec = torch.empty_like(lse)
        dqkv = torch.empty_like(qkv)
        st = native.stream_ptr()

        def fwd():
            native.check(L.vqb_attn_fwd_hd(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), N, T, C, hd, st), "fwd")

        def bwd():
            native.check(L.vqb_attn_bwd_hd(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                                           dvec.data_ptr(), dqkv.data_ptr(), N, T, C, hd, st), "bwd")

        ours_f = event_ms(fwd, a.steps, a.warmup)
        ours_b = event_ms(bwd, a.steps, a.warmup)

        qs = qkv.detach().clone().requires_grad_(True)
        q, k, v = (u.view(N, T, heads, hd).transpose(1, 2) for u in qs.chunk(3, -1))
        do = dout.view(N, T, heads, hd).transpose(1, 2)
        with torch.no_grad():
            sdpa_f = event_ms(lambda: F.scaled_dot_product_attention(q, k, v), a.steps, a.warmup)
        o = F.scaled_dot_product_attention(q, k, v)
        sdpa_b = event_ms(lambda: torch.autograd.grad(o, qs, do, retain_graph=True), a.steps, a.warmup)

        flop_f, flop_b = 4.0 * N * heads * T * T * hd, 10.0 * N * heads * T * T * hd
        print(json.dumps({
            "head_dim": hd, "heads": heads, "tokens": T, "batch": N,
            "fwd_ms": round(ours_f, 4), "fwd_sdpa_ms": round(sdpa_f, 4), "fwd_vs_sdpa": round(ours_f / sdpa_f, 3),
            "bwd_ms": round(ours_b, 4), "bwd_sdpa_ms": round(sdpa_b, 4), "bwd_vs_sdpa": round(ours_b / sdpa_b, 3),
            "fwd_tflops": round(flop_f / ours_f / 1e9, 1), "bwd_tflops": round(flop_b / ours_b / 1e9, 1),
            "sdpa_fwd_tflops": round(flop_f / sdpa_f / 1e9, 1), "sdpa_bwd_tflops": round(flop_b / sdpa_b / 1e9, 1),
            "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
