"""Times the image autoencoder's training step (vae_trainer.Trainer.step: encoder, decoder, LPIPS, optional PatchGAN
and VQ, both optimizers, as one CUDA-graph replay after the warm-up) without and with ResnetBlock recomputation
(Trainer(..., recompute=True), ae.enable_recompute).

Usage: python tools/train_mem_bench.py [--res 256] [--batch 8] [--ch 128] [--ch-mult 1,2,4,4] [--gan] [--hr] [--vq]
           [--steps 5] [--warmup 5]

Prints one JSON line per arm (plain, recompute) with ms/step, images/s and the peak allocated memory over the whole run
(warm-up, capture and timed replays), plus the card's name and power limit read in the same run. Every line also
carries the arm's saved-activation bytes predicted from the shapes (saved_activation_bytes). An arm whose prediction
exceeds 3/4 of the card's memory is not run (its line says so): the rest is left for weights, optimizer state, LPIPS,
the discriminator and the backward's transient buffers, and a run that would exhaust the card measures nothing.

The Trainer encodes 256x256 images (it area-resizes larger ones, as the reference does), so its reconstruction is
256x256, or 512x512 with --hr; --res is that reconstruction size. For any other --res both arms are reported as not
run, with the prediction for an autoencoder that encodes and decodes at --res.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "vqgan-training_b200"))
sys.path.insert(1, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

ENC_RES = 256  # what Trainer.step feeds the encoder


def saved_activation_bytes(ch, ch_mult, num_res_blocks, z_channels, hr, N, enc_res, dec_res, recompute):
    """Bytes of the activations the VAE's training forward keeps for the backward (bf16, channels padded to 8), each
    tensor counted once, by the module that saves it: conv_in, Downsample and Upsample their input; a ResnetBlock x,
    hn, h and h2 and two [N, 32, 2] fp32 GroupNorm records (recompute: x and the two records); norm_out + conv_out x
    and hn. The encoder sees enc_res x enc_res; the decoder (with hr: one more level, ch_mult + [4]) upsamples to
    dec_res x dec_res. Not counted: the latent-sized tensors, attention (the Trainer's default has none), LPIPS and the
    discriminator, which are the same in both arms."""
    cp = lambda c: -(-c // 8) * 8  # noqa: E731

    def act(c, px):
        return 2 * cp(c) * px * N

    def block(cin, cout, px):
        records = 2 * N * 32 * 2 * 4
        if recompute:
            return act(cin, px) + records
        return 2 * act(cin, px) + 2 * act(cout, px) + records

    n = len(ch_mult)
    px = enc_res * enc_res
    tot = act(3, px)  # encoder conv_in
    cin = ch
    for i in range(n):
        cout = ch * ch_mult[i]
        for _ in range(num_res_blocks):
            tot += block(cin, cout, px)
            cin = cout
        if i != n - 1:
            tot += act(cin, px)  # Downsample input
            px //= 4
    tot += 2 * block(cin, cin, px) + 2 * act(cin, px)  # mid, norm_out + conv_out
    dm = list(ch_mult) + ([4] if hr else [])
    px = (dec_res >> (len(dm) - 1)) ** 2
    cin = ch * dm[-1]
    tot += act(z_channels, px) + 2 * block(cin, cin, px)  # decoder conv_in, mid
    for i in reversed(range(len(dm))):
        cout = ch * dm[i]
        for _ in range(num_res_blocks + 1):
            tot += block(cin, cout, px)
            cin = cout
        if i != 0:
            tot += act(cin, px)  # Upsample input
            px *= 4
    return tot + 2 * act(cin, px)  # norm_out + conv_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=256, help="reconstruction size: 256, or 512 with --hr")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--ch", type=int, default=128)
    ap.add_argument("--ch-mult", default="1,2,4,4")
    ap.add_argument("--gan", action="store_true", help="PatchGAN discriminator with LeCam (hinge)")
    ap.add_argument("--hr", action="store_true", help="decoder_also_perform_hr: one more decoder level")
    ap.add_argument("--vq", action="store_true", help="VQ codebook bottleneck")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5, help="untimed steps: 3 eager ones, then the graph capture")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "train_mem_bench.py needs a CUDA (sm_90a) device: there is no CPU path"

    import vae_trainer as vt
    from infer_bench import card

    mult = [int(v) for v in a.ch_mult.split(",")]
    N = a.batch
    trainable = a.res == (2 * ENC_RES if a.hr else ENC_RES)
    enc_res = ENC_RES if trainable else a.res
    info = card()
    budget = 0.75 * torch.cuda.get_device_properties(torch.cuda.current_device()).total_memory

    for arm, recompute in (("plain", False), ("recompute", True)):
        pred = saved_activation_bytes(a.ch, mult, 2, 16, a.hr, N, enc_res, a.res, recompute)
        line = {"arm": arm, "res": a.res, "batch": N, "ch": a.ch, "ch_mult": a.ch_mult, "gan": a.gan, "hr": a.hr,
                "vq": a.vq, "predicted_saved_gb": round(pred / 2 ** 30, 2)}
        if not trainable:
            line["skipped"] = (f"Trainer.step encodes {ENC_RES}x{ENC_RES} images: its reconstruction is "
                               f"{ENC_RES}x{ENC_RES}, or {2 * ENC_RES}x{2 * ENC_RES} with --hr")
        elif pred > budget:
            line["skipped"] = f"predicted saved activations exceed 3/4 of the card ({budget / 2 ** 30:.1f} GB)"
        else:
            tr = None
            try:
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                tr = vt.Trainer("cuda", vae_ch=a.ch, vae_ch_mult=a.ch_mult, decoder_also_perform_hr=a.hr,
                                do_clamp=True, do_ganloss=a.gan, disc_type="hinge", use_lecam=a.gan, use_vq=a.vq,
                                max_steps=10 ** 6, recompute=recompute)
                batch = next(iter(vt.SyntheticLoader(N, a.res)))[0]
                for _ in range(a.warmup):
                    tr.step(batch)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    out = tr.step(batch)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / a.steps
                line.update(ms_per_step=round(ms, 2), images_per_s=round(N * 1e3 / ms, 2),
                            peak_alloc_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                            cuda_graph=tr.graph_launches_per_step is not None,
                            loss=round(float(out["overall_vae_loss"]), 5))
            except torch.OutOfMemoryError:
                line["skipped"] = "out of memory"
            finally:
                if tr is not None:
                    tr.release_graph()
                del tr
                torch.cuda.empty_cache()
        print(json.dumps(dict(line, gpu=info)), flush=True)


if __name__ == "__main__":
    main()
