#!/usr/bin/env python
"""Inference benchmark: images/s of the no-grad encoder / decoder (the reference model card's use of a trained
checkpoint), eagerly launched and replayed as one CUDA graph, beside the eager PyTorch peer on the same GPU.

    python tools/infer_bench.py --infer decode --res 768x512 --batch 4 --dtype bf16
    python tools/infer_bench.py --infer reconstruct --res 768 --ch 256 --attn --dump-outputs DIR

--res is HxW (or one number for a square image), divisible by the encoder's downsampling factor (8 for ch_mult
1,2,4,4). Weights are seeded (seeded.fill_state_dict), the input a seeded uniform image in [-1, 1) or, for
--infer decode, a seeded latent. The peer runs the same weights through the oracle restatement of the reference's
encoder_forward / decoder_forward in bf16 with cuDNN (cudnn.benchmark on): the model card's `.bfloat16()` arithmetic.
Prints one JSON line: images/s graphed and eagerly launched, peak allocated memory, the peer, and the card's name and
power limit read in the same run. --dump-outputs DIR writes the graphed run's outputs as float32 DIR/<name>.npy.

--frames T times the video autoencoder (tae.TVAE, ch_mult 1,2,4,4, num_res_blocks 2, z_channels 16) on a
(batch, 3, T, res, res) clip instead, for example

    python tools/infer_bench.py --frames 48 --res 256 --ch 64 --infer reconstruct --dtype bf16

T, H and W must be divisible by 8. reconstruct is TVAE.forward (encoder, the sampling DiagonalGaussian, decoder); the
CUDA graph captures its torch.randn_like too. The peer is oracle/tae_oracle.py in bf16 with cuDNN (cudnn.benchmark on).
The line reports videos/s and frames/s, and the forward's algorithmic FLOPs counted from the plan shapes
(tae_oracle.flops: convs with the folded up-sampling, attention matmuls), so that "tflops_per_s" is a whole-forward
rate, not a kernel's.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
sys.path.insert(1, ROOT)
os.environ.setdefault("VQB_OFFLINE", "1")

import torch  # noqa: E402


def card():
    """Name, power limit and max SM clock of the current GPU (read-only nvidia-smi query)."""
    idx = torch.cuda.current_device()
    info = {"name": torch.cuda.get_device_name(idx)}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, plim, clk = [c.strip() for c in r.stdout.strip().split(",")]
        info.update(name=name, power_limit=plim, max_sm_clock=clk)
    except Exception as e:  # the measurement stays valid; the line says what could not be read
        info["power_limit"] = f"unavailable ({type(e).__name__})"
    return info


def parse_res(s):
    h, _, w = s.lower().partition("x")
    return int(h), int(w or h)


def timed(fn, steps, warmup):
    """-> (ms per call, peak allocated bytes during the timed calls); CUDA events around `steps` calls after warm-up."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated(), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--infer", choices=["encode", "decode", "reconstruct"], default="reconstruct")
    ap.add_argument("--res", default="256", help="HxW of the image (one number: square)")
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--dtype", choices=["bf16", "fp32"], default="bf16", help="dtype of the module's parameters")
    ap.add_argument("--attn", action="store_true", help="mid-block attention (use_attn=True)")
    ap.add_argument("--ch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-eager", action="store_true", help="skip the PyTorch peer")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR")
    ap.add_argument("--frames", type=int, default=0, help="time the video autoencoder (tae.TVAE) on T frames")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "infer_bench.py needs a CUDA (sm_90a) device: there is no CPU path"
    if args.frames:
        return video_main(args)

    import ae
    import ops
    from oracle import seeded
    from oracle import vae_oracle as VO

    H, W = parse_res(args.res)
    B = args.batch
    cfg = VO.VAEConfig(resolution=256, ch=args.ch, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=16,
                       use_attn=args.attn)
    f = 2 ** (len(cfg.ch_mult) - 1)
    if H % f or W % f:
        raise SystemExit(f"--res {H}x{W}: both sides must be divisible by {f}")
    dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float32
    vae = ae.VAE(resolution=256, in_channels=3, ch=cfg.ch, out_ch=3, ch_mult=list(cfg.ch_mult),
                 num_res_blocks=cfg.num_res_blocks, z_channels=cfg.z_channels, use_attn=cfg.use_attn,
                 decoder_also_perform_hr=False, use_wavelet=False)
    tag = f"infer_bench/ch{cfg.ch}"
    sd = seeded.fill_state_dict(vae.state_dict(), tag)
    vae.load_state_dict(sd)
    vae = vae.cuda().to(dtype).eval()
    x = (seeded.tensor(tag + "/x", (B, 3, H, W), 1.0, "uniform")).cuda().to(dtype)
    zin = (seeded.tensor(tag + "/z", (B, cfg.z_channels, H // f, W // f), 1.0)).cuda().to(dtype)

    def ours():
        if args.infer == "encode":
            return {"z": vae.encoder(x).clamp(-8.0, 8.0)}
        if args.infer == "decode":
            return {"image": vae.decoder(zin)}
        z = vae.encoder(x).clamp(-8.0, 8.0)
        return {"z": z, "image": vae.decoder(z)}

    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        ops.fat_conv_enabled()  # one-time first-layer self-check, before any capture
        ms_eager, peak_eager, _ = timed(ours, args.steps, args.warmup)  # also fills the pack caches
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ours()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = ours()
        ms_graph, _, _ = timed(lambda: graph.replay(), args.steps, args.warmup)
    if args.dump_outputs:
        import numpy as np

        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in static.items():
            np.save(os.path.join(args.dump_outputs, k + ".npy"), v.detach().float().cpu().numpy())

    line = {"metric": "images/sec", "unit": "images/s", "infer": args.infer, "dtype": args.dtype,
            "config": {"ch": cfg.ch, "ch_mult": list(cfg.ch_mult), "num_res_blocks": cfg.num_res_blocks,
                       "z_channels": cfg.z_channels, "use_attn": cfg.use_attn, "res": [H, W], "batch": B},
            "value": B / (ms_graph * 1e-3), "ms_per_call_graph": ms_graph,
            "eager_launch": {"value": B / (ms_eager * 1e-3), "ms_per_call": ms_eager},
            # peak allocated memory of the eagerly launched forward (weights and inputs included); a graph replay
            # reuses the capture's private pool instead
            "peak_mem_gib": peak_eager / 2 ** 30, "weights_and_inputs_gib": base / 2 ** 30,
            "gpu": card()}
    del graph, static
    if not args.no_eager:
        sdb = {k: v.cuda().bfloat16() for k, v in sd.items()}
        xb, zb = x.bfloat16(), zin.bfloat16()
        torch.backends.cudnn.benchmark = True

        def peer():
            if args.infer == "encode":
                return VO.encoder_forward(sdb, xb, cfg).clamp(-8.0, 8.0)
            if args.infer == "decode":
                return VO.decoder_forward(sdb, zb, cfg)
            return VO.decoder_forward(sdb, VO.encoder_forward(sdb, xb, cfg).clamp(-8.0, 8.0), cfg)

        try:
            with torch.no_grad():
                ms_p, peak_p, _ = timed(peer, args.steps, args.warmup)
            line["eager_peer"] = {"value": B / (ms_p * 1e-3), "ms_per_call": ms_p, "peak_mem_gib": peak_p / 2 ** 30,
                                  "impl": "oracle encoder_forward / decoder_forward (reference arithmetic) in bf16, "
                                          "cuDNN, cudnn.benchmark=True, no autocast"}
            line["vs_eager_peer"] = line["value"] / line["eager_peer"]["value"]
        except torch.OutOfMemoryError:
            line["eager_peer"] = {"unavailable": "out of memory"}
    print(json.dumps(line), flush=True)


def video_main(args):
    import tae
    from oracle import seeded
    from oracle import tae_oracle as TO

    H, W = parse_res(args.res)
    T, B = args.frames, args.batch
    cfg = TO.TAEConfig(ch=args.ch, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=16, resolution=256)
    f = 2 ** (len(cfg.ch_mult) - 1)
    if T % f or H % f or W % f:
        raise SystemExit(f"--frames {T} --res {H}x{W}: T, H and W must be divisible by {f}")
    dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float32
    vae = tae.TVAE(**cfg.kwargs())
    tag = f"infer_bench/tae_ch{cfg.ch}"
    sd = seeded.fill_state_dict(vae.state_dict(), tag)
    vae.load_state_dict(sd)
    vae = vae.cuda().to(dtype).eval()
    x = seeded.tensor(tag + "/x", (B, 3, T, H, W), 1.0, "uniform").cuda().to(dtype)
    zin = seeded.tensor(tag + "/z", (B, cfg.z_channels, T // f, H // f, W // f), 1.0).cuda().to(dtype)

    def ours():
        if args.infer == "encode":
            return {"z": vae.encoder(x)}
        if args.infer == "decode":
            return {"video": vae.decoder(zin)}
        decz, z = vae(x)
        return {"z": z, "video": decz}

    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        ms_eager, peak_eager, _ = timed(ours, args.steps, args.warmup)  # also fills the pack caches
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ours()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = ours()
        ms_graph, _, _ = timed(lambda: graph.replay(), args.steps, args.warmup)
    if args.dump_outputs:
        import numpy as np

        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in static.items():
            np.save(os.path.join(args.dump_outputs, k + ".npy"), v.detach().float().cpu().numpy())
    flops = TO.flops(cfg, B, T, H, W, args.infer)
    line = {"metric": "videos/sec", "unit": "videos/s", "model": "tae.TVAE", "infer": args.infer, "dtype": args.dtype,
            "config": {"ch": cfg.ch, "ch_mult": list(cfg.ch_mult), "num_res_blocks": cfg.num_res_blocks,
                       "z_channels": cfg.z_channels, "frames": T, "res": [H, W], "batch": B},
            "value": B / (ms_graph * 1e-3), "frames_per_s": B * T / (ms_graph * 1e-3), "ms_per_call_graph": ms_graph,
            "eager_launch": {"value": B / (ms_eager * 1e-3), "frames_per_s": B * T / (ms_eager * 1e-3),
                             "ms_per_call": ms_eager},
            "algorithmic_tflop": flops / 1e12, "tflops_per_s_graph": flops / (ms_graph * 1e-3) / 1e12,
            "peak_mem_gib": peak_eager / 2 ** 30, "weights_and_inputs_gib": base / 2 ** 30,
            "gpu": card()}
    del graph, static
    if not args.no_eager:
        sdb = {k: v.cuda().bfloat16() for k, v in sd.items()}
        xb, zb = x.bfloat16(), zin.bfloat16()
        torch.backends.cudnn.benchmark = True

        def peer():
            if args.infer == "encode":
                return TO.encoder_forward(sdb, xb, cfg)
            if args.infer == "decode":
                return TO.decoder_forward(sdb, zb, cfg)
            z = TO.encoder_forward(sdb, xb, cfg)
            return TO.decoder_forward(sdb, TO.reg(z, torch.randn_like(z.chunk(2, 1)[0])), cfg), z

        try:
            with torch.no_grad():
                ms_p, peak_p, _ = timed(peer, args.steps, args.warmup)
            line["eager_peer"] = {"value": B / (ms_p * 1e-3), "frames_per_s": B * T / (ms_p * 1e-3),
                                  "ms_per_call": ms_p, "peak_mem_gib": peak_p / 2 ** 30,
                                  "tflops_per_s": flops / (ms_p * 1e-3) / 1e12,
                                  "impl": "oracle tae_oracle encoder_forward / reg / decoder_forward (reference "
                                          "arithmetic: literal nearest-x2 + conv3d) in bf16, cuDNN, "
                                          "cudnn.benchmark=True, no autocast"}
            line["vs_eager_peer"] = line["value"] / line["eager_peer"]["value"]
        except torch.OutOfMemoryError:
            line["eager_peer"] = {"unavailable": "out of memory"}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
