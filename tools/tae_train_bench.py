"""Times one training step of the video autoencoder (tae.TVAE opted in with tae.enable_training): forward, backward and
torch.optim.AdamW, against the same step of the reference arithmetic (oracle/tae_oracle.py: F.conv3d, F.group_norm,
softmax attention) under bf16 autocast with cuDNN on the same GPU.

Usage: python tools/tae_train_bench.py [--frames 16] [--res 256] [--ch 64] [--batch 1] [--steps 5] [--warmup 2]
           [--skip-peer]

Prints one JSON line per arm (native, peer) with steps/s, frames/s, whole-step TFLOP/s and peak allocated memory, plus
the card's name and power limit read in the same run. FLOPs are counted from the plan shapes (step_flops): the forward
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--ch", type=int, default=64)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-peer", action="store_true")
    a = ap.parse_args()

    import tae

    cfg = TO.TAEConfig(ch=a.ch)
    N, T, H, W = a.batch, a.frames, a.res, a.res
    flops = step_flops(cfg, N, T, H, W)
    info = card()
    torch.manual_seed(0)
    x = torch.rand(N, 3, T, H, W, device="cuda") * 2 - 1

    def report(arm, ms, peak):
        print(json.dumps({"arm": arm, "frames": T, "res": a.res, "ch": a.ch, "batch": N, "ms_per_step": round(ms, 2),
                          "steps_per_s": round(1e3 / ms, 3), "frames_per_s": round(N * T * 1e3 / ms, 2),
                          "tflops": round(flops / ms / 1e9, 1), "peak_alloc_gb": round(peak / 2 ** 30, 2),
                          "gpu": info}), flush=True)

    torch.manual_seed(1)
    vae = tae.enable_training(tae.TVAE(**cfg.kwargs()).cuda())
    opt = torch.optim.AdamW(vae.parameters(), lr=1e-4)

    def native_step():
        opt.zero_grad(set_to_none=True)
        decz, z = vae(x)
        loss = _loss(decz, x, z)
        loss.backward()
        opt.step()
        return loss

    ms, peak, _ = timed(native_step, a.steps, a.warmup)
    report("native", ms, peak)
    del vae, opt
    torch.cuda.empty_cache()
    if a.skip_peer:
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
    report("bf16-autocast cuDNN peer", ms, peak)


if __name__ == "__main__":
    main()
