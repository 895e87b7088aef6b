"""Training of the video autoencoder (tae.TVAE) against the image autoencoder's loss stack, applied per frame, in one
process or data-parallel over ranks.

The reference has no video trainer. A clip [B, 3, T, H, W] is scored by the reference image losses on its frames folded
into the batch in (b, t) order (DESIGN.md section 7): LPIPS and the PatchGAN discriminator see the B*T' frames of the
selection as one image batch, and GradNorm normalises the gradient of the whole clip. utils.LPIPS and
utils.PatchDiscriminator take the clip directly (ops.ClipToFrames): no folded copy of the clip is made.

    tr = VideoTrainer(tae.TVAE(...).cuda(), utils.LPIPS().cuda(), utils.PatchDiscriminator().cuda(),
                      disc_type="hinge", use_lecam=True, perceptual_frames=4, lr_vae=1e-4, lr_disc=2e-4)
    out = tr.step(clip)        # clip: fp32 [B, 3, T, H, W] on cuda

Every term above scores frames one at a time. `clip_discriminator=tae_disc.PatchDiscriminator3D(...)` adds a 3-D
PatchGAN that convolves over time as well: its D step runs after the per-frame one on the whole clip (real: the clip,
fake: the detached reconstruction; `perceptual_frames` does not apply), with the same loss type and LeCam but its own
anchors and AdamW, and the G pass adds its generator loss on gradnorm(decz, clip_disc_weight).

Data parallel, as the image Trainer (vae_trainer.py): when a process group of more than one rank exists, each rank
trains on its own clips and the TVAE and discriminator gradients are averaged over ranks (one all-reduce each on the
flat gradient buffer of FlatAdamW), the LeCam anchors are fed by rank-averaged logits, GradNorm divides by the
rank-averaged norm, and LPIPS scores with rank 0's weights. The torchrun entry point (`train_video`, below):

    torchrun --nproc_per_node=8 tae_trainer.py --vae_ch 64 --clip_frames 16 --resolution 256 --batch_size 1 \
        --do_ganloss --disc_type hinge --use_lecam True --perceptual_frames 4 [--do_clip_ganloss]

Out of scope: CUDA-graph capture (the step runs eagerly), the latent flip and crop augmentations, HR decoding of the
image Trainer, and real video datasets (the entry point trains on a seeded synthetic clip stream).
"""
from __future__ import annotations

import logging
import os
import sys
import time

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import click
import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

import tae
from flat import FlatAdamW, check_ema_decay
from utils import broadcast_module_state
from vae_trainer import (FlatAllReduceDDP, SyntheticLoader, _dist_on, avg_scalar_over_nodes, cleanup,
                         cosine_with_warmup, gan_disc_loss, gradnorm, restart_ema, vae_loss_function)


EVAL_SEED = 20040101  # seed of train_video's held-out clips (--eval_clips), fixed across runs and ranks


def fold_frames(x: torch.Tensor, frames=None) -> torch.Tensor:
    """[B, C, T, H, W] -> [B*T', C, H, W] in (b, t) order (frames: [B, T'] selection, None = every frame). An ATen
    copy, for the terms that take images rather than clips (the MSE of the lpips=None baseline)."""
    B, C, T, H, W = x.shape
    if frames is None:
        return x.transpose(1, 2).reshape(B * T, C, H, W)
    if x.is_cuda:  # pinned + non_blocking: a pageable host-to-device copy would wait for the stream to drain
        frames = frames.pin_memory().to(x.device, non_blocking=True)
    idx = frames.reshape(B, -1, 1, 1, 1).expand(-1, -1, C, H, W)
    return torch.gather(x.transpose(1, 2), 1, idx).reshape(-1, C, H, W)


class VideoTrainer:
    """Trainer._step_body (vae_trainer.py) on frames folded into the batch, in one process or data-parallel.

    vae: a float32 tae.TVAE; it is opted into training here (tae.enable_training; `recompute` passes through).
    lpips: utils.LPIPS (frozen; its train/eval mode is kept as given), or None for the MSE-only baseline, whose
        reconstruction term is F.mse_loss over the selected frames instead of the gradnormed LPIPS mean.
    discriminator: utils.PatchDiscriminator or None (no GAN terms). disc_type "hinge" or "bce"; use_lecam adds the
        LeCam regulariser with the anchors of Trainer (weight 0.1, EMA 0.9).
    perceptual_frames: k draws k distinct frames per clip per step from torch's CPU generator (torch.manual_seed makes
        runs reproducible); LPIPS, the MSE term and both GAN passes use that one selection. None: every frame.
    lr_vae, lr_disc: learning rates of the fused AdamW (vqb_adamw_flat; betas (0.9, 0.95), weight decay 1e-3, as in
        Trainer) over the TVAE and the discriminator.
    clip_discriminator: tae_disc.PatchDiscriminator3D or None; it is opted into training here. lr_clip_disc: its AdamW
        learning rate (same betas and weight decay); clip_disc_weight: the GradNorm weight of its generator pass.
    ema_decay: None, or 0 < d < 1 to keep an exponential moving average of the TVAE's trained weights in its fused
        AdamW launch (flat.FlatAdamW; not of the discriminators). `vae_ema` is a tae.TVAE over the average (None
        without one); evaluate(clips, ema=True) scores it.

    step(clip) per step:
      1. decz, z = vae(clip) (the reparameterisation draws its noise from torch's CUDA generator);
      2. with a discriminator: D on real and detached fake frames, hinge / BCE loss (+ LeCam), AdamW step of D;
      3. with a clip discriminator D3: D3 on the whole real and detached fake clip, the same loss (+ LeCam with the
         clip_lecam_anchor_{real,fake}_logits), AdamW step of D3;
      4. LPIPS(gradnorm(decz), clip).mean() over the selected frames, vae_loss_function(clip, gradnorm(decz, 0.001),
         z) with z the NCTHW encoder output (0.1 * mean(z^2)), the generator loss of D on gradnorm(decz, 1.0) with
         D's parameters frozen for that pass, and that of D3 on gradnorm(decz, clip_disc_weight) with D3 frozen; one
         backward, AdamW step of the TVAE.

    Data parallel (a process group of more than one rank exists when the trainer is built): the constructor wraps the
    TVAE and the discriminators in vae_trainer.FlatAllReduceDDP, which broadcasts rank 0's parameters and buffers,
    before FlatAdamW re-homes them into its flat buffers, so every cached bf16 operand is packed from rank 0's weights;
    LPIPS is broadcast from rank 0 too. Each step then averages D's (and D3's) flat gradient over ranks before its AdamW
    step and the TVAE's before the TVAE's (in place, in FlatAdamW's gradient buffer; VQB_DDP_OVERLAP as in Trainer), feeds the
    LeCam anchors with rank-averaged logits (avg_scalar_over_nodes), and GradNorm divides by the rank-averaged norm.
    Every rank therefore holds the same weights, optimizer moments and anchors after every step. Without a process
    group the wrappers issue no collective and the step is the single-process step.
    `vae`, `disc` and `clip_disc` are the unwrapped modules.

    Randomness: the frame selection comes from torch's CPU generator and ε from torch's CUDA generator, so ranks draw
    their own frames and noise when their caller seeds them per rank (train_video: torch.manual_seed(seed + rank));
    their weights agree anyway because of the constructor broadcast.
    """

    def __init__(self, vae: nn.Module, lpips, discriminator=None, *, disc_type="hinge", use_lecam=False,
                 perceptual_frames=None, lr_vae, lr_disc=None, recompute=False, clip_discriminator=None,
                 lr_clip_disc=None, clip_disc_weight=1.0, ema_decay=None):
        if ema_decay is not None:
            ema_decay = check_ema_decay(ema_decay)
        if disc_type not in ("hinge", "bce"):
            raise ValueError(f"unknown disc_type {disc_type!r}")
        if discriminator is not None and lr_disc is None:
            raise ValueError("lr_disc is required with a discriminator")
        if clip_discriminator is not None and lr_clip_disc is None:
            raise ValueError("lr_clip_disc is required with a clip discriminator")
        if perceptual_frames is not None and perceptual_frames < 1:
            raise ValueError(f"perceptual_frames must be >= 1, got {perceptual_frames}")
        self.vae = tae.enable_training(vae, recompute=recompute)
        self.lpips, self.disc = lpips, discriminator
        self.disc_type, self.use_lecam, self.perceptual_frames = disc_type, use_lecam, perceptual_frames
        # the order of Trainer.__init__: broadcast (in the wrappers' constructors) before FlatAdamW re-homes the weights
        self._vae_dp = FlatAllReduceDDP(vae)
        self._disc_dp = None
        if discriminator is not None:
            discriminator.requires_grad_(True)
            self._disc_dp = FlatAllReduceDDP(discriminator)
        self.optimizer_G = FlatAdamW([{"params": [p for p in vae.parameters() if p.requires_grad], "lr": lr_vae}],
                                     weight_decay=1e-3, betas=(0.9, 0.95), ema_decay=ema_decay)
        self._vae_dp.attach_store(self.optimizer_G.store)
        self.vae_ema = None
        if ema_decay is not None:  # started after the broadcast, from the weights every rank holds
            self.vae_ema = self.optimizer_G.averaged_copy(vae)
            self._vae_dp.after_load = lambda: restart_ema(self.optimizer_G, self.vae, self.vae_ema)
        self.optimizer_D = None
        device = next(vae.parameters()).device
        if discriminator is not None:
            self.optimizer_D = FlatAdamW([{"params": list(discriminator.parameters()), "lr": lr_disc}],
                                         weight_decay=1e-3, betas=(0.9, 0.95))
            self._disc_dp.attach_store(self.optimizer_D.store)
        if lpips is not None:
            broadcast_module_state(lpips)  # frozen, not wrapped: every rank scores with rank 0's weights
        self.lecam_loss_weight, self.lecam_beta = 0.1, 0.9
        self.lecam_anchor_real_logits = torch.zeros((), device=device)
        self.lecam_anchor_fake_logits = torch.zeros((), device=device)
        self.last_frames = None
        self.clip_disc, self._clip_disc_dp, self.optimizer_clip_D = None, None, None
        if clip_discriminator is not None:
            self.clip_disc = tae.enable_training(clip_discriminator.requires_grad_(True))
            self._clip_disc_dp = FlatAllReduceDDP(clip_discriminator)  # broadcast before FlatAdamW re-homes the weights
            self.optimizer_clip_D = FlatAdamW([{"params": list(clip_discriminator.parameters()), "lr": lr_clip_disc}],
                                              weight_decay=1e-3, betas=(0.9, 0.95))
            self._clip_disc_dp.attach_store(self.optimizer_clip_D.store)
            self.clip_disc_weight = clip_disc_weight
            self.clip_lecam_anchor_real_logits = torch.zeros((), device=device)
            self.clip_lecam_anchor_fake_logits = torch.zeros((), device=device)

    def draw_frames(self, B: int, T: int):
        """[B, k] int64 CPU tensor of k distinct frames per clip (torch's CPU generator), or None for every frame."""
        k = self.perceptual_frames
        if k is None:
            return None
        if k > T:
            raise ValueError(f"perceptual_frames={k} exceeds the clip's {T} frames")
        return torch.stack([torch.randperm(T)[:k] for _ in range(B)])

    def step(self, clip: torch.Tensor) -> dict:
        if clip.dim() != 5 or clip.shape[1] != 3:
            raise ValueError(f"expected a [B, 3, T, H, W] clip, got shape {tuple(clip.shape)}")
        sel = self.draw_frames(clip.shape[0], clip.shape[2])
        self.last_frames = sel
        vae_dp, disc_dp = self._vae_dp, self._disc_dp
        disc = None if disc_dp is None else disc_dp.module
        decz, z = vae_dp.module(clip)

        out = {}
        if disc is not None:
            real_preds = disc(clip, frames=sel)
            fake_preds = disc(decz.detach(), frames=sel)
            d_loss, avg_real_logits, avg_fake_logits, disc_acc = gan_disc_loss(real_preds, fake_preds, self.disc_type)
            if _dist_on():  # one process uses the local means as they are: no copy is launched
                avg_real_logits = avg_scalar_over_nodes(avg_real_logits, clip.device)
                avg_fake_logits = avg_scalar_over_nodes(avg_fake_logits, clip.device)
            self.lecam_anchor_real_logits.mul_(self.lecam_beta).add_(avg_real_logits, alpha=1 - self.lecam_beta)
            self.lecam_anchor_fake_logits.mul_(self.lecam_beta).add_(avg_fake_logits, alpha=1 - self.lecam_beta)
            total_d_loss = d_loss.mean()
            out["d_loss"] = total_d_loss.detach()
            lecam_loss_item = torch.zeros((), device=clip.device)
            if self.use_lecam:
                lecam_loss = (real_preds - self.lecam_anchor_fake_logits).pow(2).mean() + \
                    (fake_preds - self.lecam_anchor_real_logits).pow(2).mean()
                lecam_loss_item = lecam_loss.detach()
                total_d_loss = total_d_loss + lecam_loss * self.lecam_loss_weight
            self.optimizer_D.zero_grad(set_to_none=True)
            total_d_loss.backward()
            disc_dp.allreduce_grads()
            self.optimizer_D.step()
            out.update(avg_real_logits=avg_real_logits, avg_fake_logits=avg_fake_logits, disc_acc=disc_acc,
                       lecam_loss=lecam_loss_item)
        if self.clip_disc is not None:
            out.update(self._clip_disc_step(clip, decz))

        if self.lpips is not None:
            recon_loss = self.lpips(gradnorm(decz), clip, frames=sel).mean()
        else:
            recon_loss = F.mse_loss(fold_frames(decz, sel), fold_frames(clip, sel))
        # at its defaults (do_recon=False, as in Trainer) vae_loss_function reads only z: the images it would compare,
        # the selected frames of clip and of gradnorm(decz, 0.001), are passed as the clips they fold from
        vae_loss, loss_data = vae_loss_function(clip, gradnorm(decz, weight=0.001), z)
        overall_vae_loss = recon_loss + vae_loss
        if disc is not None:
            disc.requires_grad_(False)  # the G pass needs D's data gradient only
            try:
                fake_preds = disc(gradnorm(decz, weight=1.0), frames=sel)
            finally:
                disc.requires_grad_(True)
            if self.disc_type == "bce":
                g_gan_loss = F.binary_cross_entropy_with_logits(fake_preds, torch.ones_like(fake_preds))
            else:
                g_gan_loss = -fake_preds.mean()
            overall_vae_loss = overall_vae_loss + g_gan_loss
            out["g_gan_loss"] = g_gan_loss.detach()
        if self.clip_disc is not None:
            clip_disc = self.clip_disc
            clip_disc.requires_grad_(False)  # the G pass needs D3's data gradient only
            try:
                fake_preds = clip_disc(gradnorm(decz, weight=self.clip_disc_weight))
            finally:
                clip_disc.requires_grad_(True)
            if self.disc_type == "bce":
                clip_g_gan_loss = F.binary_cross_entropy_with_logits(fake_preds, torch.ones_like(fake_preds))
            else:
                clip_g_gan_loss = -fake_preds.mean()
            overall_vae_loss = overall_vae_loss + clip_g_gan_loss
            out["clip_g_gan_loss"] = clip_g_gan_loss.detach()

        self.optimizer_G.zero_grad(set_to_none=True)
        overall_vae_loss.backward()
        vae_dp.allreduce_grads()
        self.optimizer_G.step()
        out.update(overall_vae_loss=overall_vae_loss.detach(), perceptual_loss=recon_loss.detach(),
                   loss_data=loss_data, z=z.detach(), reconstructed=decz.detach())
        return out

    def _clip_disc_step(self, clip, decz) -> dict:
        """The D step of the clip discriminator on the whole clip (real: clip, fake: decz.detach()), with its own LeCam
        anchors and AdamW; the same loss as the per-frame D step."""
        real_preds = self.clip_disc(clip)
        fake_preds = self.clip_disc(decz.detach())
        d_loss, avg_real_logits, avg_fake_logits, disc_acc = gan_disc_loss(real_preds, fake_preds, self.disc_type)
        if _dist_on():
            avg_real_logits = avg_scalar_over_nodes(avg_real_logits, clip.device)
            avg_fake_logits = avg_scalar_over_nodes(avg_fake_logits, clip.device)
        self.clip_lecam_anchor_real_logits.mul_(self.lecam_beta).add_(avg_real_logits, alpha=1 - self.lecam_beta)
        self.clip_lecam_anchor_fake_logits.mul_(self.lecam_beta).add_(avg_fake_logits, alpha=1 - self.lecam_beta)
        total_d_loss = d_loss.mean()
        out = {"clip_d_loss": total_d_loss.detach()}
        lecam_loss_item = torch.zeros((), device=clip.device)
        if self.use_lecam:
            lecam_loss = (real_preds - self.clip_lecam_anchor_fake_logits).pow(2).mean() + \
                (fake_preds - self.clip_lecam_anchor_real_logits).pow(2).mean()
            lecam_loss_item = lecam_loss.detach()
            total_d_loss = total_d_loss + lecam_loss * self.lecam_loss_weight
        self.optimizer_clip_D.zero_grad(set_to_none=True)
        total_d_loss.backward()
        self._clip_disc_dp.allreduce_grads()
        self.optimizer_clip_D.step()
        out.update(clip_avg_real_logits=avg_real_logits, clip_avg_fake_logits=avg_fake_logits,
                   clip_disc_acc=disc_acc, clip_lecam_loss=lecam_loss_item)
        return out

    @torch.no_grad()
    def evaluate(self, clips, ema=False) -> dict:
        """Reconstruction quality of held-out clips: `clips` is an iterable of fp32 [B, 3, T, H, W] clips in [-1, 1).

        Each clip is encoded by the TVAE and its posterior mean (the first half of the encoder's channels; nothing is
        sampled, so a checkpoint's score does not depend on the RNG) decoded. The frames are scored with
        ops.psnr_ssim(decz, clip, value_range=(-1, 1)) and, when the trainer has an LPIPS, with
        lpips(decz.clamp(-1, 1), clip) in eval mode (dropout off; its previous mode is restored).

        Returns psnr, ssim (and lpips) as Python floats, the means over every frame, and psnr_frames, ssim_frames (and
        lpips_frames) as fp32 [N, T] tensors, N the clips' batch rows in order. Weights, packed operands, optimizer
        moments, LeCam anchors, module modes and RNG states are left as they were, and no collective is issued.
        ema=True scores the averaged weights (vae_ema) instead of the trained ones."""
        import ops

        if ema and self.vae_ema is None:
            raise ValueError("evaluate(ema=True): this trainer keeps no weight EMA (ema_decay=None)")
        vae, lpips = (self.vae_ema if ema else self.vae), self.lpips
        was_training = lpips.training if lpips is not None else None
        scores = {"psnr": [], "ssim": [], "lpips": []}
        try:
            if lpips is not None:
                lpips.eval()
            for clip in clips:
                if clip.dim() != 5 or clip.shape[1] != 3:
                    raise ValueError(f"expected [B, 3, T, H, W] clips, got shape {tuple(clip.shape)}")
                z = vae.encoder(clip)
                decz = vae.decoder(z[:, :z.shape[1] // 2])
                p, s = ops.psnr_ssim(decz, clip, value_range=(-1.0, 1.0))
                scores["psnr"].append(p)
                scores["ssim"].append(s)
                if lpips is not None:
                    scores["lpips"].append(lpips(decz.clamp(-1, 1), clip).view(p.shape))
        finally:
            if lpips is not None:
                lpips.train(was_training)
        if not scores["psnr"]:
            raise ValueError("evaluate: no clips")
        out = {}
        for k, v in scores.items():
            if v:
                frames = torch.cat(v)
                out[k] = float(frames.double().mean())
                out[f"{k}_frames"] = frames
        return out


@click.command()
@click.option("--batch_size", type=int, default=1, help="Clips per rank per step")
@click.option("--clip_frames", type=int, default=16, help="Frames per clip")
@click.option("--resolution", type=int, default=256, help="Height and width of the clips")
@click.option("--perceptual_frames", type=int, default=None,
              help="Frames per clip the losses score each step, drawn at random (default: every frame)")
@click.option("--do_ganloss", is_flag=True, help="Whether to use GAN loss")
@click.option("--disc_type", type=click.Choice(["bce", "hinge"]), default="bce", help="Discriminator type")
@click.option("--use_lecam", type=bool, default=False, help="Whether to use Lecam")
@click.option("--no_lpips", is_flag=True, help="Train with the MSE of the scored frames instead of LPIPS")
@click.option("--recompute", is_flag=True, help="Recompute ResnetBlock activations in the backward (less memory)")
@click.option("--learning_rate_vae", type=float, default=1e-4, help="Learning rate for the TVAE")
@click.option("--learning_rate_disc", type=float, default=2e-4, help="Learning rate for discriminator")
@click.option("--vae_ch", type=int, default=64, help="Base channel size for the TVAE")
@click.option("--vae_ch_mult", type=str, default="1,2,4,4", help="Channel multipliers for the TVAE")
@click.option("--vae_num_res_blocks", type=int, default=2, help="Number of residual blocks for the TVAE")
@click.option("--vae_z_channels", type=int, default=16, help="Number of latent channels for the TVAE")
@click.option("--max_steps", type=int, default=1000, help="Maximum number of steps to train for")
@click.option("--evaluate_every_n_steps", type=int, default=250, help="Save a checkpoint every n steps")
@click.option("--load_path", type=str, default=None, help="TVAE state_dict to start from (a saved checkpoint)")
@click.option("--run_name", type=str, default="run", help="Checkpoints are saved under ./ckpt/<run_name>/")
@click.option("--seed", type=int, default=42, help="Rank r seeds torch with seed + r (frame selection and noise)")
@click.option("--do_clip_ganloss", is_flag=True, help="Also train against a 3-D PatchGAN on whole clips (tae_disc)")
@click.option("--clip_disc_ch", type=int, default=64, help="Base channels of the clip discriminator (multiple of 32)")
@click.option("--clip_disc_layers", type=int, default=3, help="Stride-2 layers of the clip discriminator")
@click.option("--learning_rate_clip_disc", type=float, default=None,
              help="Learning rate for the clip discriminator (default: --learning_rate_disc)")
@click.option("--eval_clips", type=int, default=0,
              help="Held-out clips rank 0 reconstructs and scores (PSNR, SSIM, LPIPS) at every checkpoint (0: none)")
@click.option("--ema_decay", type=float, default=None,
              help="Keep an EMA of the TVAE weights with this decay (0 < D < 1, warmed up over the first updates) and "
                   "save it beside every checkpoint (default: none)")
def train_video(batch_size, clip_frames, resolution, perceptual_frames, do_ganloss, disc_type, use_lecam, no_lpips,
                recompute, learning_rate_vae, learning_rate_disc, vae_ch, vae_ch_mult, vae_num_res_blocks,
                vae_z_channels, max_steps, evaluate_every_n_steps, load_path, run_name, seed, do_clip_ganloss,
                clip_disc_ch, clip_disc_layers, learning_rate_clip_disc, eval_clips, ema_decay):
    """Trains tae.TVAE on a seeded synthetic clip stream, data-parallel under torchrun (one process per GPU, NCCL) or in
    one process. Rank 0 logs every 5 steps and saves the TVAE's state_dict every --evaluate_every_n_steps steps; with
    --eval_clips K it first scores K held-out clips (VideoTrainer.evaluate) and logs eval_psnr, eval_ssim and
    eval_lpips. With --ema_decay D it also saves the averaged weights as tvae_ema_step_<k>.pt (a TVAE state_dict) and,
    with --eval_clips, logs eval_ema_psnr, eval_ema_ssim and eval_ema_lpips."""
    # arguments are checked before anything touches a device
    if ema_decay is not None and not 0.0 < ema_decay < 1.0:
        raise click.BadParameter(f"must satisfy 0 < D < 1, got {ema_decay}", param_hint="--ema_decay")
    if eval_clips < 0:
        raise click.BadParameter(f"must be >= 0, got {eval_clips}", param_hint="--eval_clips")
    if perceptual_frames is not None and not 1 <= perceptual_frames <= clip_frames:
        raise click.BadParameter(f"must be between 1 and --clip_frames ({clip_frames}), got {perceptual_frames}",
                                 param_hint="--perceptual_frames")
    try:
        ch_mult = [int(c) for c in vae_ch_mult.split(",")]
    except ValueError:
        raise click.BadParameter(f"expected comma-separated integers, got {vae_ch_mult!r}", param_hint="--vae_ch_mult")
    div = 2 ** (len(ch_mult) - 1)
    if clip_frames % div or resolution % div:
        raise click.BadParameter(f"--clip_frames ({clip_frames}) and --resolution ({resolution}) must be multiples of "
                                 f"{div} for {len(ch_mult)} levels", param_hint="--vae_ch_mult")
    extra = {}  # the clip discriminator's settings, eval_clips and ema_decay, passed only when used
    if do_clip_ganloss:
        if clip_disc_ch <= 0 or clip_disc_ch % 32 or clip_disc_ch > 256:
            raise click.BadParameter(f"must be a multiple of 32 up to 256, got {clip_disc_ch}",
                                     param_hint="--clip_disc_ch")
        if clip_disc_layers < 1:
            raise click.BadParameter(f"must be >= 1, got {clip_disc_layers}", param_hint="--clip_disc_layers")
        f = 2 ** clip_disc_layers
        if clip_frames % f or resolution % f:
            raise click.BadParameter(f"--clip_frames ({clip_frames}) and --resolution ({resolution}) must be multiples "
                                     f"of {f} for {clip_disc_layers} layers", param_hint="--clip_disc_layers")
        lr = learning_rate_disc if learning_rate_clip_disc is None else learning_rate_clip_disc
        extra["clip_disc"] = (clip_disc_ch, clip_disc_layers, lr)
    if eval_clips:
        extra["eval_clips"] = eval_clips
    if ema_decay is not None:
        extra["ema_decay"] = ema_decay

    assert torch.cuda.is_available(), "CUDA is required"
    rank = int(os.environ.get("RANK", "0"))
    device = torch.device(f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}")
    torch.cuda.set_device(device)
    if "RANK" in os.environ:
        dist.init_process_group(backend="nccl", device_id=device)
    try:
        _train_video(rank, device, batch_size, clip_frames, resolution, perceptual_frames, do_ganloss, disc_type,
                     use_lecam, no_lpips, recompute, learning_rate_vae, learning_rate_disc, vae_ch, ch_mult,
                     vae_num_res_blocks, vae_z_channels, max_steps, evaluate_every_n_steps, load_path, run_name, seed,
                     **extra)
    finally:
        cleanup()


def _train_video(rank, device, batch_size, clip_frames, resolution, perceptual_frames, do_ganloss, disc_type, use_lecam,
                 no_lpips, recompute, learning_rate_vae, learning_rate_disc, vae_ch, ch_mult, vae_num_res_blocks,
                 vae_z_channels, max_steps, evaluate_every_n_steps, load_path, run_name, seed, clip_disc=None,
                 eval_clips=0, ema_decay=None):
    """clip_disc: (ch, n_layers, learning rate) of a tae_disc.PatchDiscriminator3D to train against, or None.
    eval_clips: the number of held-out clips rank 0 scores at every checkpoint.
    ema_decay: keep a weight EMA (VideoTrainer) and save it, and score it, at every checkpoint; None: no EMA."""
    import tae_disc
    import utils

    torch.manual_seed(seed + rank)  # each rank draws its own frames and noise (the weights come from rank 0)
    torch.cuda.manual_seed(seed + rank)
    vae = tae.TVAE(resolution=resolution, in_channels=3, ch=vae_ch, out_ch=3, ch_mult=ch_mult,
                   num_res_blocks=vae_num_res_blocks, z_channels=vae_z_channels)
    if load_path is not None:
        vae.load_state_dict(torch.load(load_path, map_location="cpu"), strict=True)
    lpips = None if no_lpips else utils.LPIPS().to(device)  # train mode: dropout live, as train_ddp runs it
    disc = utils.PatchDiscriminator().to(device) if do_ganloss else None
    clip_kw = {}
    if clip_disc is not None:
        ch, n_layers, lr = clip_disc
        clip_kw = dict(clip_discriminator=tae_disc.PatchDiscriminator3D(ch=ch, n_layers=n_layers).to(device),
                       lr_clip_disc=lr)
    tr = VideoTrainer(vae.to(device), lpips, disc, disc_type=disc_type, use_lecam=use_lecam,
                      perceptual_frames=perceptual_frames, lr_vae=learning_rate_vae, lr_disc=learning_rate_disc,
                      recompute=recompute, ema_decay=ema_decay, **clip_kw)
    lr_scheduler = cosine_with_warmup(tr.optimizer_G, 200, max_steps)
    clips = iter(SyntheticLoader(batch_size, resolution, frames=clip_frames))  # seed 42 + rank
    held_out = []
    if eval_clips and rank == 0:  # the same clips on every run, whatever --seed: scores compare across runs
        held_out = SyntheticLoader(1, resolution, seed=EVAL_SEED, n_distinct=eval_clips, frames=clip_frames).batches

    logger = logging.getLogger(__name__)
    logger.setLevel(logging.INFO)
    if rank == 0:
        handler = logging.StreamHandler()
        handler.setFormatter(logging.Formatter("%(asctime)s - %(name)s - %(levelname)s - %(message)s"))
        logger.addHandler(handler)
    t_log, step_log = time.time(), 0
    for step in range(max_steps):
        out = tr.step(next(clips)[0].to(device, non_blocking=True))
        lr_scheduler.step()
        if rank == 0 and step % 5 == 0:  # the only host synchronisations of the loop
            ld = out["loss_data"]
            items = [("overall_vae_loss", out["overall_vae_loss"]), ("perceptual_loss", out["perceptual_loss"]),
                     ("kl_loss", ld["kl_loss"])]
            if do_ganloss:
                items += [("d_loss", out["d_loss"]), ("gan_loss", out["g_gan_loss"]),
                          ("avg_real_logits", out["avg_real_logits"]), ("avg_fake_logits", out["avg_fake_logits"]),
                          ("discriminator_accuracy", out["disc_acc"]), ("lecam_loss", out["lecam_loss"]),
                          ("lecam_anchor_real_logits", tr.lecam_anchor_real_logits),
                          ("lecam_anchor_fake_logits", tr.lecam_anchor_fake_logits)]
            if clip_disc is not None:
                items += [("clip_d_loss", out["clip_d_loss"]), ("clip_gan_loss", out["clip_g_gan_loss"]),
                          ("clip_avg_real_logits", out["clip_avg_real_logits"]),
                          ("clip_avg_fake_logits", out["clip_avg_fake_logits"]),
                          ("clip_discriminator_accuracy", out["clip_disc_acc"]),
                          ("clip_lecam_loss", out["clip_lecam_loss"])]
            items = [(k, float(v)) for k, v in items]
            now = time.time()
            items.append(("ms_per_step", (now - t_log) * 1e3 / (step + 1 - step_log)))
            t_log, step_log = now, step + 1
            logger.info(f"step {step} - " + "\n\t".join(f"{k}: {v:.4f}" for k, v in items))
        if evaluate_every_n_steps > 0 and (step + 1) % evaluate_every_n_steps == 0 and rank == 0:
            if held_out:
                ev = tr.evaluate(c.to(device, non_blocking=True) for c in held_out)
                logger.info(f"step {step + 1} - " + "\n\t".join(f"eval_{k}: {ev[k]:.4f}" for k in
                                                                  ("psnr", "ssim", "lpips") if k in ev))
                if tr.vae_ema is not None:
                    ev = tr.evaluate((c.to(device, non_blocking=True) for c in held_out), ema=True)
                    logger.info(f"step {step + 1} - " + "\n\t".join(f"eval_ema_{k}: {ev[k]:.4f}" for k in
                                                                      ("psnr", "ssim", "lpips") if k in ev))
            os.makedirs(f"./ckpt/{run_name}", exist_ok=True)
            ck = f"./ckpt/{run_name}/tvae_step_{step + 1}.pt"
            torch.save({k: v.detach().cpu() for k, v in tr.vae.state_dict().items()}, ck)
            logger.info(f"Saved checkpoint to {ck}")
            if tr.vae_ema is not None:  # the averaged weights, loadable by --load_path and tae.TVAE.load_state_dict
                ck = f"./ckpt/{run_name}/tvae_ema_step_{step + 1}.pt"
                torch.save({k: v.detach().cpu() for k, v in tr.vae_ema.state_dict().items()}, ck)
                logger.info(f"Saved checkpoint to {ck}")


if __name__ == "__main__":
    # Example: torchrun --nproc_per_node=8 tae_trainer.py --vae_ch 64 --clip_frames 16 --resolution 256 --batch_size 1
    train_video()
