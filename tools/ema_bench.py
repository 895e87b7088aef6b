"""Cost of the weight EMA fused into the AdamW launch (vqb_adamw_ema_flat_dev, flat.FlatAdamW(ema_decay=...)), in one
run, each leg with and without the average, the two arms alternated round by round so that drift of the shared card
hits both alike:

  optimizer  the launch alone over the flat buffer of the FLUX-config VAE (ch=128, ch_mult 1,2,4,4, two res blocks, z 16):
             ms per launch (CUDA events over --launches launches per round after a warm-up), GB/s of the compulsory
             traffic counted from the shapes (AdamW reads p, g, m, v and writes p, m, v: 28 B per element; the EMA
             reads and writes e: 36 B) and its share of the H100 SXM's 3.35 TB/s
  trainer    vae_trainer.Trainer.step at --batch x 256^2 (the bench.py `lpips` config), CUDA-graph replay
  video      tae_trainer.VideoTrainer.step on one 1 x 3 x 16 x 256^2 clip, TVAE ch=64 (LPIPS on every frame, no GAN)

Usage: python tools/ema_bench.py [--rounds 5] [--launches 200] [--steps 10] [--batch 32] [--skip-trainers]
One JSON line per leg, each with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
sys.path.insert(1, ROOT)
sys.path.insert(2, os.path.join(ROOT, "tools"))
os.environ.setdefault("VQB_OFFLINE", "1")

import torch  # noqa: E402

from infer_bench import card  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data-sheet HBM3 bandwidth (700 W card)
DECAY = 0.999
FLUX = dict(resolution=256, in_channels=3, ch=128, out_ch=3, ch_mult=[1, 2, 4, 4], num_res_blocks=2, z_channels=16)


def events_ms(fn, n):
    """ms per call of `fn`, CUDA events around n calls."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternated(arms, rounds, n, warmup):
    """{name: [ms per call of each round]}: every arm warmed up, then `rounds` rounds of n calls per arm, in turn."""
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    out = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            out[k].append(events_ms(fn, n))
    return out


def summary(ms):
    return {"median_ms": round(statistics.median(ms), 4), "min_ms": round(min(ms), 4), "max_ms": round(max(ms), 4)}


def optimizer_leg(info, a):
    import ae
    from flat import CHUNK, FlatAdamW

    arms, opts = {}, {}
    for name, decay in (("plain", None), ("ema", DECAY)):
        torch.manual_seed(0)
        vae = ae.VAE(use_attn=False, decoder_also_perform_hr=False, use_wavelet=False, **FLUX).cuda()
        opt = FlatAdamW([{"params": list(vae.parameters()), "lr": 1e-4}], weight_decay=1e-3, betas=(0.9, 0.95),
                        ema_decay=decay)
        opt.store.grads.normal_()
        active = (True,) * len(opt.store.plist)
        opt.upload_hyper(active)  # one record; the launches below re-read it (the EMA count does not matter for time)
        opts[name] = (vae, opt)
        arms[name] = lambda opt=opt, active=active: opt.launch(active)
    n = opts["plain"][1].store.total
    res = alternated(arms, a.rounds, a.launches, warmup=20)
    line = {"leg": "optimizer", "elements": n, "chunks": n // CHUNK, "launches_per_round": a.launches,
            "rounds": a.rounds}
    for name, per_elem in (("plain", 28), ("ema", 36)):
        s = summary(res[name])
        gbs = per_elem * n / (s["median_ms"] * 1e6)
        s.update(bytes=per_elem * n, GB_per_s=round(gbs, 1), share_of_3_35TB_s=round(gbs / (HBM_TBS * 1e3), 3))
        line[name] = s
    line["ema_minus_plain_ms"] = round(line["ema"]["median_ms"] - line["plain"]["median_ms"], 4)
    line.update(gpu=info["name"], power_limit=info["power_limit"])
    print(json.dumps(line), flush=True)


def trainer_leg(info, a):
    import vae_trainer as vt

    arms, keep = {}, []
    for name, decay in (("plain", None), ("ema", DECAY)):
        tr = vt.Trainer("cuda:0", vae_resolution=256, vae_ch=128, vae_ch_mult="1,2,4,4", vae_num_res_blocks=2,
                        vae_z_channels=16, do_clamp=True, max_steps=10 ** 6, lpips_eval=True, cuda_graph=True,
                        ema_decay=decay)
        g = torch.Generator().manual_seed(1)
        batch = (torch.rand(a.batch, 3, 256, 256, generator=g) * 2 - 1).pin_memory()
        keep.append(tr)
        arms[name] = lambda tr=tr, batch=batch: tr.step(batch)
    res = alternated(arms, a.rounds, a.steps, warmup=tr.GRAPH_WARMUP_STEPS + 2)
    line = {"leg": "Trainer.step", "batch": a.batch, "res": 256, "ch": 128, "graph_replay": True,
            "steps_per_round": a.steps, "rounds": a.rounds,
            "launches_per_replay": {k: t.graph_launches_per_step for k, t in zip(arms, keep)}}
    for name in arms:
        line[name] = summary(res[name])
    line["ema_minus_plain_ms"] = round(line["ema"]["median_ms"] - line["plain"]["median_ms"], 3)
    line.update(gpu=info["name"], power_limit=info["power_limit"])
    print(json.dumps(line), flush=True)
    for tr in keep:
        tr.release_graph()


def video_leg(info, a):
    import tae
    import tae_trainer
    import utils

    arms = {}
    clip = torch.rand(1, 3, 16, 256, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)) * 2 - 1
    for name, decay in (("plain", None), ("ema", DECAY)):
        torch.manual_seed(0)
        vae = tae.TVAE(resolution=256, in_channels=3, ch=64, out_ch=3, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
                       z_channels=16).cuda()
        tr = tae_trainer.VideoTrainer(vae, utils.LPIPS().cuda(), None, lr_vae=1e-4, ema_decay=decay)
        arms[name] = lambda tr=tr: tr.step(clip)
    res = alternated(arms, a.rounds, max(2, a.steps // 2), warmup=2)
    line = {"leg": "VideoTrainer.step", "clip": [1, 3, 16, 256, 256], "ch": 64, "rounds": a.rounds}
    for name in arms:
        line[name] = summary(res[name])
    line["ema_minus_plain_ms"] = round(line["ema"]["median_ms"] - line["plain"]["median_ms"], 3)
    line.update(gpu=info["name"], power_limit=info["power_limit"])
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200, help="optimizer launches per arm per round (>= 100)")
    ap.add_argument("--steps", type=int, default=10, help="trainer steps per arm per round")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--skip-trainers", action="store_true", help="time the optimizer launch only")
    a = ap.parse_args()
    if a.launches < 100:
        ap.error("--launches must be >= 100")
    assert torch.cuda.is_available(), "the measurement needs a CUDA device"
    info = card()
    print(json.dumps({"card": info}), flush=True)
    optimizer_leg(info, a)
    torch.cuda.empty_cache()
    if not a.skip_trainers:
        trainer_leg(info, a)
        torch.cuda.empty_cache()
        video_leg(info, a)


if __name__ == "__main__":
    main()
