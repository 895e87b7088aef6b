"""Tiled against untiled encode / decode of the video autoencoder (tiling.encode / tiling.decode, vqb_tile_blend), with
the TVAE at --ch (default 64, ch_mult 1,2,4,4, two res blocks, z 16) in --dtype (default bf16), seeded random weights:

  clip     decode and reconstruct (encode + decode) of a 1 x 3 x --frames x --res^2 clip (default 48 x 512^2), tiled
           with --tile / --overlap (default (16, 256, 256) / (8, 64, 64)) and untiled
  1080p    decode of z [1, 16, 15, 136, 240] (a 120 x 1088 x 1920 clip) with tile (48, 512, 512), overlap (8, 64, 64),
           tiled only

Each arm: ms per call (CUDA events around --steps calls after --warmup calls), frames/s and peak allocated memory. Each
tiled leg also prints the plan's recompute factor prod(n L / X) over the axes. The clip legs print the time in their
blend launches (the torch profiler's device time of tile_blend_kernel in one separate call) in ms, as a share of the
tiled call and in GB/s of the traffic counted from the shapes (tile read, accumulator read where a tile is not the
first, accumulator write, the bf16 output written once) against 3.35 TB/s. The untiled arm runs only when its peak
predicted from the shapes is at most 3/4 of the card; when both run the line carries their max abs difference (a
consistency figure with random weights, not a quality claim). One JSON line per leg, with the card's name and power
limit read in the same run.

Usage: python tools/tiled_bench.py [--frames 48] [--res 512] [--ch 64] [--dtype bf16] [--steps 3] [--warmup 1]
       [--skip-1080p]   (the 1080p leg times one call after one warm-up call and does not profile its blend)
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
sys.path.insert(1, ROOT)
sys.path.insert(2, os.path.join(ROOT, "tools"))
os.environ.setdefault("VQB_OFFLINE", "1")

import torch  # noqa: E402

from infer_bench import card  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data-sheet HBM3 bandwidth (700 W card)


def events_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        y = fn()
        del y
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated() - base


def predicted_untiled_peak(ch, ch_mult, voxels, out_bytes):
    """No-grad peak of an untiled decode / reconstruct from the shapes: the first full-resolution ResnetBlock of the
    decoder holds its upsampled bf16 NTHWC input at ch*ch_mult[1] channels and its normalised copy, plus two
    ch*ch_mult[0]-channel tensors (conv1 output and the shortcut), at every output voxel; plus the output."""
    return voxels * 2 * (2 * ch * ch_mult[1] + 2 * ch * ch_mult[0]) + out_bytes


def plan_stats(axes, n_ch, tile_es, out_bf16):
    """(recompute factor, blend bytes) of a decode plan, counted from the shapes."""
    recompute = math.prod(a.n * a.glen / a.gextent for a in axes)
    grid = n_ch * math.prod(a.gextent for a in axes)
    tile_elems = n_ch * math.prod(a.n * a.glen for a in axes)
    nbytes = tile_elems * (tile_es + 4) + (tile_elems - grid) * 4 + (grid * 2 if out_bf16 else 0)
    return recompute, nbytes


def blend_ms(fn):
    """Device time of the tile_blend_kernel launches in one call of fn, from the torch profiler."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "tile_blend_kernel" in e.key)
    return us / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--ch", type=int, default=64)
    ap.add_argument("--dtype", choices=["bf16", "fp32"], default="bf16")
    ap.add_argument("--tile", type=int, nargs=3, default=[16, 256, 256])
    ap.add_argument("--overlap", type=int, nargs=3, default=[8, 64, 64])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--skip-1080p", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tiled_bench.py measures on a CUDA device; none is present")

    import tae
    import tiling
    from oracle import seeded

    dev = card()
    dt = torch.bfloat16 if a.dtype == "bf16" else torch.float32
    ch_mult = [1, 2, 4, 4]
    m = tae.TVAE(resolution=256, in_channels=3, ch=a.ch, out_ch=3, ch_mult=ch_mult, num_res_blocks=2, z_channels=16)
    m.load_state_dict(seeded.fill_state_dict(m.state_dict(), "tiled_bench"))
    m = m.cuda().to(dt).eval()
    f = tiling.factor(m.decoder)
    budget = 0.75 * torch.cuda.get_device_properties(0).total_memory
    es = 2 if dt == torch.bfloat16 else 4

    def leg(name, x, latent, run_tiled, run_untiled, frames, tile, overlap, n_out_ch, steps, warmup, profile=True):
        line = {"leg": name, "input": list(x.shape), "dtype": a.dtype, "ch": a.ch, "tile": tile, "overlap": overlap,
                **dev}
        axes = [tiling._Axis(X, L, O, f, True) for X, L, O in zip(latent, tile, overlap)]  # the decode's plan
        recompute, nbytes = plan_stats(axes, n_out_ch, es, dt == torch.bfloat16)
        voxels = math.prod(ax.gextent for ax in axes)
        pred = predicted_untiled_peak(a.ch, ch_mult, voxels, voxels * n_out_ch * es)
        with torch.no_grad():
            ms, peak = events_ms(run_tiled, steps, warmup)
            bms = blend_ms(run_tiled) if profile else 0.0
            line.update(tiled_ms=round(ms, 2), tiled_frames_per_s=round(frames * 1000 / ms, 2),
                        tiled_peak_gb=round(peak / 2 ** 30, 2), recompute_factor=round(recompute, 3),
                        blend_ms=round(bms, 3) if profile else "not measured",
                        blend_share=round(bms / ms, 5) if profile else "not measured",
                        blend_gbs=round(nbytes / bms / 1e6, 1) if bms > 0 else None,
                        blend_share_of_hbm=round(nbytes / bms / 1e6 / (HBM_TBS * 1e3), 3) if bms > 0 else None,
                        predicted_untiled_peak_gb=round(pred / 2 ** 30, 2))
            if run_untiled is None:
                pass
            elif pred > budget:
                line["untiled"] = f"not run: predicted peak {pred / 2 ** 30:.1f} GB exceeds 3/4 of the card"
            else:
                ums, upeak = events_ms(run_untiled, steps, warmup)
                diff = (run_tiled().float() - run_untiled().float()).abs().max().item()
                line.update(untiled_ms=round(ums, 2), untiled_frames_per_s=round(frames * 1000 / ums, 2),
                            untiled_peak_gb=round(upeak / 2 ** 30, 2), time_ratio=round(ms / ums, 3),
                            max_abs_diff=diff)
        print(json.dumps(line), flush=True)

    tile, overlap = list(a.tile), list(a.overlap)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.rand(1, 3, a.frames, a.res, a.res, device="cuda", generator=g) * 2 - 1).to(dt)
    z = torch.randn(1, 16, a.frames // f, a.res // f, a.res // f, device="cuda", generator=g).to(dt)
    lat = tuple(z.shape[2:])
    leg("clip decode", z, lat, lambda: tiling.decode(m.decoder, z, tile=tile, overlap=overlap), lambda: m.decoder(z),
        a.frames, tile, overlap, 3, a.steps, a.warmup)

    def recon_tiled():
        mom = tiling.encode(m.encoder, x, tile=tile, overlap=overlap)
        return tiling.decode(m.decoder, mom[:, :16].contiguous(), tile=tile, overlap=overlap)

    def recon_untiled():
        return m.decoder(m.encoder(x)[:, :16].contiguous())

    leg("clip reconstruct", x, lat, recon_tiled, recon_untiled, a.frames, tile, overlap, 3, a.steps, a.warmup)
    del x, z
    if not a.skip_1080p:
        z = torch.randn(1, 16, 15, 136, 240, device="cuda", generator=g).to(dt)
        t8, o8 = [48, 512, 512], [8, 64, 64]
        # one timed call after one warm-up call: a call is 45 tile forwards; the blend share is taken on the clip legs
        leg("1080p decode", z, tuple(z.shape[2:]), lambda: tiling.decode(m.decoder, z, tile=t8, overlap=o8), None, 120,
            t8, o8, 3, 1, 1, profile=False)


if __name__ == "__main__":
    main()
