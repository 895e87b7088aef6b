"""Times tae_trainer.VideoTrainer.step (the video autoencoder trained against per-frame losses) for three loss stacks:
MSE only (lpips=None), + LPIPS, and + LPIPS + PatchGAN (hinge, LeCam), each on every frame of the clip and on
--perceptual-frames frames per clip. Every arm is also run as a bf16-autocast eager peer: the same folded computation
in plain PyTorch (oracle/tae_oracle.py, oracle/clip_loss_oracle.py: F.conv3d / F.conv2d VGG16 with cuDNN) with
torch.optim.AdamW.

With --clip-disc it times instead the 3-D PatchGAN leg: LPIPS + clip discriminator (tae_disc.PatchDiscriminator3D,
--clip-disc-ch 64, --clip-disc-layers 3, hinge + LeCam) on every frame, without and with the per-frame PatchGAN, and
the peer with the oracle module (oracle/clip_disc_oracle.py, F.conv3d on cuDNN); it also prints the discriminator's
FLOPs counted from the plan shapes.

Usage: python tools/tae_loss_bench.py [--frames 16] [--res 256] [--ch 64] [--batch 1] [--perceptual-frames 4]
           [--steps 5] [--warmup 2] [--skip-peer] [--clip-disc [--clip-disc-ch 64] [--clip-disc-layers 3]]

Prints one JSON line per arm with ms/step, frames/s (clip frames through the autoencoder per second) and peak
allocated memory, plus the card's name and power limit read in the same run. LPIPS / PatchD weights are torchvision's
random initialisation (VQB_OFFLINE=1): the timing does not depend on the values.
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
import torch.nn.functional as F  # noqa: E402

from infer_bench import card, timed  # noqa: E402
from oracle import clip_disc_oracle as CDO  # noqa: E402
from oracle import clip_loss_oracle as CO  # noqa: E402
from oracle import loss_oracle as LO  # noqa: E402
from oracle import tae_oracle as TO  # noqa: E402

STACKS = ("mse", "lpips", "lpips+gan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--ch", type=int, default=64)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--perceptual-frames", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-peer", action="store_true")
    ap.add_argument("--clip-disc", action="store_true")
    ap.add_argument("--clip-disc-ch", type=int, default=64)
    ap.add_argument("--clip-disc-layers", type=int, default=3)
    a = ap.parse_args()

    import tae
    import tae_disc
    import tae_trainer
    import utils

    cfg = TO.TAEConfig(ch=a.ch)
    N, T = a.batch, a.frames
    info = card()
    torch.manual_seed(0)
    x = torch.rand(N, 3, T, a.res, a.res, device="cuda") * 2 - 1
    torch.manual_seed(1)
    tsd = tae.TVAE(**cfg.kwargs()).state_dict()
    lsd = utils.LPIPS().state_dict()
    psd = utils.PatchDiscriminator().state_dict()
    nl = a.clip_disc_layers
    csd = CDO.PatchDiscriminator3D(ch=a.clip_disc_ch, n_layers=nl).state_dict()

    def report(arm, stack, k, ms, peak):
        print(json.dumps({"arm": arm, "loss": stack, "perceptual_frames": k or T, "frames": T, "res": a.res,
                          "ch": a.ch, "batch": N, "ms_per_step": round(ms, 2),
                          "frames_per_s": round(N * T * 1e3 / ms, 1), "peak_alloc_gb": round(peak / 2 ** 30, 2),
                          "gpu": info}), flush=True)

    def native(stack, k):
        m = tae.TVAE(**cfg.kwargs())
        m.load_state_dict(tsd)
        lp = pd = d3 = None
        if stack != "mse":
            lp = utils.LPIPS()
            lp.load_state_dict(lsd)
            lp = lp.cuda().eval()
        if stack.startswith("lpips+gan"):
            pd = utils.PatchDiscriminator()
            pd.load_state_dict(psd)
            pd = pd.cuda()
        if stack.endswith("clipd"):
            d3 = tae_disc.PatchDiscriminator3D(ch=a.clip_disc_ch, n_layers=nl)
            d3.load_state_dict(csd)
            d3 = d3.cuda()
        tr = tae_trainer.VideoTrainer(m.cuda(), lp, pd, disc_type="hinge", use_lecam=True, perceptual_frames=k,
                                      lr_vae=1e-4, lr_disc=2e-4, clip_discriminator=d3, lr_clip_disc=2e-4)
        ms, peak, _ = timed(lambda: tr.step(x), a.steps, a.warmup)
        report("native", stack, k, ms, peak)
        del tr, m, lp, pd, d3
        torch.cuda.empty_cache()

    def peer(stack, k):
        tp = {n: v.cuda().clone().requires_grad_(True) for n, v in tsd.items()}
        ls = {n: v.cuda() for n, v in lsd.items()}
        dp = {n: v.cuda().clone().requires_grad_("scaling_layer" not in n) for n, v in psd.items()}
        kw = dict(weight_decay=1e-3, betas=(0.9, 0.95))
        opt_g = torch.optim.AdamW(tp.values(), lr=1e-4, **kw)
        opt_d = torch.optim.AdamW([v for v in dp.values() if v.requires_grad], lr=2e-4, **kw)
        anchors = [torch.zeros((), device="cuda"), torch.zeros((), device="cuda")]
        cp = {n: v.cuda().clone().requires_grad_(True) for n, v in csd.items()}
        opt_c = torch.optim.AdamW(cp.values(), lr=2e-4, **kw)
        canchors = [torch.zeros((), device="cuda"), torch.zeros((), device="cuda")]

        def d_step(fwd, params, opt, anc, fake_in):
            with ac():
                real, fake = fwd(params, x).float(), fwd(params, fake_in).float()
            d_loss = (F.relu(1 - real).mean() + F.relu(1 + fake).mean()) * 0.5
            anc[0] = 0.9 * anc[0] + 0.1 * real.detach().mean()
            anc[1] = 0.9 * anc[1] + 0.1 * fake.detach().mean()
            d_loss = d_loss + 0.1 * LO.lecam_loss(real, fake, anc[0], anc[1])
            opt.zero_grad(set_to_none=True)
            d_loss.backward()
            opt.step()
        ac = lambda: torch.autocast("cuda", dtype=torch.bfloat16)  # noqa: E731

        def step():
            sel = None if k is None else torch.stack([torch.randperm(T)[:k] for _ in range(N)])
            with ac():
                z = TO.encoder_forward(tp, x, cfg)
                decz = TO.decoder_forward(tp, TO.reg(z, torch.randn_like(z[:, :cfg.z_channels])), cfg)
            decz, z = decz.float(), z.float()
            patchd = lambda p, v: CO.patchd_clip(p, v, sel)  # noqa: E731
            clipd = lambda p, v: CDO.forward(p, v, nl)  # noqa: E731
            if stack.startswith("lpips+gan"):
                d_step(patchd, dp, opt_d, anchors, decz.detach())
            if stack.endswith("clipd"):
                d_step(clipd, cp, opt_c, canchors, decz.detach())
            with ac():
                if stack == "mse":
                    rec = F.mse_loss(CO.fold_frames(decz, sel), CO.fold_frames(x, sel))
                else:
                    rec = CO.lpips_clip(ls, LO.gradnorm(decz), x, sel).float().mean()
                loss = rec + 0.1 * z.pow(2).mean()
                if stack.startswith("lpips+gan"):
                    frozen = {n: v.detach() for n, v in dp.items()}
                    loss = loss - CO.patchd_clip(frozen, LO.gradnorm(decz, 1.0), sel).float().mean()
                if stack.endswith("clipd"):
                    frozen = {n: v.detach() for n, v in cp.items()}
                    loss = loss - CDO.forward(frozen, LO.gradnorm(decz, 1.0), nl).float().mean()
            opt_g.zero_grad(set_to_none=True)
            loss.backward()
            opt_g.step()
            return loss

        ms, peak, _ = timed(step, a.steps, a.warmup)
        report("bf16-autocast eager peer", stack, k, ms, peak)
        del tp, dp, opt_g, opt_d, cp, opt_c
        torch.cuda.empty_cache()

    if a.clip_disc:
        # one forward of D3 per clip; a step runs it 3 times (real, fake, G pass), the weight gradient twice (real and
        # fake of the D step) and the data gradient of every conv but conv_in twice and of all convs once (G pass)
        fwd = CDO.flops(a.clip_disc_ch, nl, N, T, a.res, a.res)
        first = CDO.flops(a.clip_disc_ch, nl, N, T, a.res, a.res, only_first=True)
        print(json.dumps({"clip_disc": {"ch": a.clip_disc_ch, "n_layers": nl, "fwd_gflop": round(fwd / 1e9, 2),
                                        "step_gflop": round((3 * fwd + 2 * fwd + 2 * (fwd - first) + fwd) / 1e9, 2)},
                          "gpu": info}), flush=True)
        for stack in ("lpips+clipd", "lpips+gan+clipd"):
            native(stack, None)
            if not a.skip_peer:
                peer(stack, None)
        return
    for k in (None, a.perceptual_frames):
        for stack in STACKS:
            native(stack, k)
            if not a.skip_peer:
                peer(stack, k)


if __name__ == "__main__":
    main()
