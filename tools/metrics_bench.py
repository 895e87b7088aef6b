"""Times ops.psnr_ssim (the fused PSNR / SSIM kernel, csrc/metrics.cu) on images and clips, beside an eager PyTorch
peer of the same definition (oracle/metrics_oracle.psnr_ssim_torch: the float32 map, then the separable window as
per-plane F.conv2d on cuDNN in float32), and VideoTrainer.evaluate on one clip beside one VideoTrainer.step.

Usage: python tools/metrics_bench.py [--steps 50] [--warmup 10] [--skip-eval]

Cases: 8 x 3 x 256^2 images, 1 x 3 x 16 x 256^2 and 1 x 3 x 48 x 256^2 clips, each in fp32 and bf16 (the peer reads
the same tensors). Per case one JSON line: ms per call (CUDA events over --steps calls after --warmup), GB/s of the
compulsory traffic (x and y read once) and its share of the H100 SXM's 3.35 TB/s, and the FLOP the definition needs,
counted from the shapes (flop() below). The evaluation leg times VideoTrainer.evaluate on one 1 x 3 x 16 x 256^2 clip
(TVAE ch=64, ch_mult 1,2,4,4, two res blocks, z 16; LPIPS) beside one step of the same trainer (LPIPS on every frame,
no GAN). The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
sys.path.insert(1, ROOT)
sys.path.insert(2, os.path.join(ROOT, "tools"))
os.environ.setdefault("VQB_OFFLINE", "1")

import torch  # noqa: E402

from infer_bench import card, timed  # noqa: E402
from oracle import metrics_oracle as MO  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data-sheet HBM3 bandwidth (700 W card)
CASES = [("image", (8, 3, 256, 256)), ("clip16", (1, 3, 16, 256, 256)), ("clip48", (1, 3, 48, 256, 256))]


def flop(shape):
    """Arithmetic of the definition per (b, c, t) plane, separable window: the value map (2 x 3 per value), the three
    products and the squared difference (3 + 3 per value), the horizontal pass over H rows and the vertical pass over
    H - 10 rows (5 moments x 11 taps x 2 per position) and the SSIM formula (~20 per valid position)."""
    H, W = shape[-2:]
    planes = 1
    for d in shape[:-2]:
        planes *= d
    Ho, Wo = H - 10, W - 10
    return planes * (12 * H * W + 2 * 11 * 5 * (H * Wo + Ho * Wo) + 20 * Ho * Wo)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--skip-eval", action="store_true", help="skip the VideoTrainer.evaluate leg")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the measurement needs a CUDA device"
    import ops

    info = card()
    print(json.dumps({"card": info}), flush=True)
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, shape in CASES:
        x32 = torch.rand(shape, device="cuda", generator=g) * 2 - 1
        y32 = (x32 + 0.1 * torch.randn(shape, device="cuda", generator=g)).clamp(-1, 1)
        for dtype in (torch.float32, torch.bfloat16):
            x, y = x32.to(dtype), y32.to(dtype)
            nbytes = 2 * x.numel() * x.element_size()
            ms, _, (p, s) = timed(lambda: ops.psnr_ssim(x, y, value_range=(-1, 1)), a.steps, a.warmup)
            ms_peer, _, (pp, sp) = timed(lambda: MO.psnr_ssim_torch(x, y, (-1, 1), torch.float32), a.steps, a.warmup)
            gbs = nbytes / ms / 1e6
            print(json.dumps({
                "case": name, "shape": list(shape), "dtype": str(dtype).split(".")[-1],
                "ms": round(ms, 4), "GB_per_s": round(gbs, 1), "share_of_3.35TB_s": round(gbs / (HBM_TBS * 1e3), 3),
                "GFLOP": round(flop(shape) / 1e9, 3), "GFLOP_per_s": round(flop(shape) / ms / 1e6, 1),
                "peer_ms": round(ms_peer, 4), "speedup_vs_peer": round(ms_peer / ms, 2),
                "max_abs_diff_vs_peer": {"psnr": float((p - pp).abs().max()), "ssim": float((s - sp).abs().max())},
                "gpu": info["name"], "power_limit": info["power_limit"]}), flush=True)
            del x, y
    if not a.skip_eval:
        evaluation_leg(info, max(2, a.steps // 10), 2)


def evaluation_leg(info, steps, warmup):
    import tae
    import tae_trainer
    import utils

    torch.manual_seed(0)
    vae = tae.TVAE(resolution=256, in_channels=3, ch=64, out_ch=3, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
                   z_channels=16).cuda()
    tr = tae_trainer.VideoTrainer(vae, utils.LPIPS().cuda(), None, lr_vae=1e-4)
    clip = torch.rand(1, 3, 16, 256, 256, device="cuda") * 2 - 1
    ms_step, mem_step, _ = timed(lambda: tr.step(clip), steps, warmup)
    ms_eval, mem_eval, ev = timed(lambda: tr.evaluate([clip]), steps, warmup)
    print(json.dumps({"case": "evaluate", "clip": [1, 3, 16, 256, 256], "ch": 64, "evaluate_ms": round(ms_eval, 2),
                      "step_ms": round(ms_step, 2), "evaluate_over_step": round(ms_eval / ms_step, 3),
                      "evaluate_peak_GB": round(mem_eval / 2 ** 30, 2), "step_peak_GB": round(mem_step / 2 ** 30, 2),
                      "psnr": round(ev["psnr"], 3), "ssim": round(ev["ssim"], 4), "lpips": round(ev["lpips"], 4),
                      "gpu": info["name"], "power_limit": info["power_limit"]}), flush=True)


if __name__ == "__main__":
    main()
