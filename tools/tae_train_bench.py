"""Times one training step of the video autoencoder (tae.TVAE opted in with tae.enable_training): forward, backward and
torch.optim.AdamW, against the same step of the reference arithmetic (oracle/tae_oracle.py: F.conv3d, F.group_norm,
softmax attention) under bf16 autocast with cuDNN on the same GPU.

Usage: python tools/tae_train_bench.py [--frames 16] [--res 256] [--ch 64] [--batch 1] [--steps 5] [--warmup 2]
           [--skip-peer] [--recompute]

Prints one JSON line per arm (native, native + recompute with --recompute, peer) with steps/s, frames/s, whole-step
TFLOP/s and peak allocated memory, plus the card's name and power limit read in the same run. Every line also carries
the arm's saved-activation bytes predicted from the shapes (saved_activation_bytes). An arm whose prediction exceeds
3/4 of the card's memory is not run (its line says so): the rest is left for weights, optimizer state and the
backward's transient buffers, and a run that would exhaust the card measures nothing.

FLOPs are counted from the plan shapes (step_flops), the same for every arm: the recompute arm's extra conv1 forwards
show up as a lower TFLOP/s. step_flops counts the forward
GEMMs of oracle.tae_oracle.flops, plus for every convolution a weight-gradient GEMM and a data-gradient GEMM of the
same size as its forward (27 rotated taps for stride 1; the 1 to 8 taps of the eight parity classes, 27 in all, over the
Downsample's output grid; 64 taps over the low-resolution grid for the folded up-sampling, as its 8 forward phases of 8),
except the data gradient of the encoder's conv_in (the video needs no gradient); the attention backward's four matmuls
(dV, dP, dQ, dK) are twice the forward's two. Elementwise, GroupNorm and softmax work is not counted.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
sys.path.insert(1, ROOT)
sys.path.insert(2, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from infer_bench import card, timed  # noqa: E402
from oracle import tae_oracle as TO  # noqa: E402


def _loss(decz, x, z):
    return F.mse_loss(decz, x) + 1e-3 * z.pow(2).mean()


def step_flops(cfg, N, T, H, W):
    """Algorithmic FLOPs of forward + backward of one training step (see the module docstring)."""
    conv_in_dgrad = 2 * cfg.in_channels * cfg.ch * 27 * T * H * W * N
    return 3 * TO.flops(cfg, N, T, H, W) - conv_in_dgrad


def saved_activation_bytes(cfg, N, T, H, W, recompute):
    """Bytes of the activations the native training forward keeps for the backward (bf16, channels padded to 8), each
    tensor counted once, by the module that saves it: conv_in, Downsample and Upsample their input; a ResnetBlock x,
    hn, h and h2 (recompute: x and two [N, 32, 2] fp32 GroupNorm records); an AttnBlock x, hn, qkv, the attention
    output and its fp32 log-sum-exp; norm_out + conv_out x and hn; the reparameterisation z and eps (fp32). A lower
    bound for the eager bf16-autocast peer, which keeps at least these tensors in at least this precision."""
    cp = lambda c: -(-c // 8) * 8  # noqa: E731
    tot = 0

    def act(c, v):
        return 2 * cp(c) * v * N

    def block(cin, cout, v):
        if recompute:
            return act(cin, v) + 2 * (N * 32 * 2 * 4)
        return act(cin, v) * 2 + act(cout, v) * 2

    def mid(c, v):
        return 2 * block(c, c, v) + act(c, v) * 6 + 4 * 8 * v * N

    n = len(cfg.ch_mult)
    ch, vox = cfg.ch, T * H * W
    tot += act(cfg.in_channels, vox)  # encoder conv_in
    cin = ch
    for i in range(n):
        cout = ch * cfg.ch_mult[i]
        for _ in range(cfg.num_res_blocks):
            tot += block(cin, cout, vox)
            cin = cout
        if i != n - 1:
            tot += act(cin, vox)  # Downsample input
            vox //= 8
    tot += mid(cin, vox) + 2 * act(cin, vox)  # mid, norm_out + conv_out
    tot += 4 * 3 * cfg.z_channels * vox * N  # z and eps
    cin = ch * cfg.ch_mult[-1]
    tot += act(cfg.z_channels, vox) + mid(cin, vox)  # decoder conv_in, mid
    for i in reversed(range(n)):
        cout = ch * cfg.ch_mult[i]
        for _ in range(cfg.num_res_blocks + 1):
            tot += block(cin, cout, vox)
            cin = cout
        if i != 0:
            tot += act(cin, vox)  # Upsample input
            vox *= 8
    return tot + 2 * act(cin, vox)  # norm_out + conv_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--ch", type=int, default=64)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-peer", action="store_true")
    ap.add_argument("--recompute", action="store_true",
                    help="also time the native step with tae.enable_training(vae, recompute=True)")
    a = ap.parse_args()

    import tae

    cfg = TO.TAEConfig(ch=a.ch)
    N, T, H, W = a.batch, a.frames, a.res, a.res
    flops = step_flops(cfg, N, T, H, W)
    info = card()
    budget = 0.75 * torch.cuda.get_device_properties(torch.cuda.current_device()).total_memory
    torch.manual_seed(0)
    x = torch.rand(N, 3, T, H, W, device="cuda") * 2 - 1

    def report(arm, ms, peak, pred):
        line = {"arm": arm, "frames": T, "res": a.res, "ch": a.ch, "batch": N,
                "predicted_saved_gb": round(pred / 2 ** 30, 2)}
        if ms is None:
            line["skipped"] = f"predicted saved activations exceed 3/4 of the card ({budget / 2 ** 30:.1f} GB)"
        else:
            line.update(ms_per_step=round(ms, 2), steps_per_s=round(1e3 / ms, 3),
                        frames_per_s=round(N * T * 1e3 / ms, 2), tflops=round(flops / ms / 1e9, 1),
                        peak_alloc_gb=round(peak / 2 ** 30, 2))
        print(json.dumps(dict(line, gpu=info)), flush=True)

    def native(arm, recompute):
        pred = saved_activation_bytes(cfg, N, T, H, W, recompute)
        if pred > budget:
            report(arm, None, None, pred)
            return
        torch.manual_seed(1)
        vae = tae.enable_training(tae.TVAE(**cfg.kwargs()).cuda(), recompute=recompute)
        opt = torch.optim.AdamW(vae.parameters(), lr=1e-4)

        def native_step():
            opt.zero_grad(set_to_none=True)
            decz, z = vae(x)
            loss = _loss(decz, x, z)
            loss.backward()
            opt.step()
            return loss

        ms, peak, _ = timed(native_step, a.steps, a.warmup)
        report(arm, ms, peak, pred)
        del vae, opt
        torch.cuda.empty_cache()

    native("native", False)
    if a.recompute:
        native("native + recompute", True)
    if a.skip_peer:
        return
    pred = saved_activation_bytes(cfg, N, T, H, W, False)  # a lower bound for the peer
    if pred > budget:
        report("bf16-autocast cuDNN peer", None, None, pred)
        return
    torch.manual_seed(1)
    sd = {k: v.cuda().requires_grad_(True) for k, v in tae.TVAE(**cfg.kwargs()).state_dict().items()}
    popt = torch.optim.AdamW(sd.values(), lr=1e-4)

    def peer_step():
        popt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            z = TO.encoder_forward(sd, x, cfg)
            eps = torch.randn_like(z[:, :cfg.z_channels])
            decz = TO.decoder_forward(sd, TO.reg(z, eps), cfg)
            loss = _loss(decz.float(), x, z.float())
        loss.backward()
        popt.step()
        return loss

    ms, peak, _ = timed(peer_step, a.steps, a.warmup)
    report("bf16-autocast cuDNN peer", ms, peak, pred)


if __name__ == "__main__":
    main()
