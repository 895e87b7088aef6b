"""Training step of the video autoencoder (tae.TVAE) against the image autoencoder's loss stack, applied per frame.

The reference has no video trainer. A clip [B, 3, T, H, W] is scored by the reference image losses on its frames folded
into the batch in (b, t) order (DESIGN.md section 7): LPIPS and the PatchGAN discriminator see the B*T' frames of the
selection as one image batch, and GradNorm normalises the gradient of the whole clip. utils.LPIPS and
utils.PatchDiscriminator take the clip directly (ops.ClipToFrames): no folded copy of the clip is made.

    tr = VideoTrainer(tae.TVAE(...).cuda(), utils.LPIPS().cuda(), utils.PatchDiscriminator().cuda(),
                      disc_type="hinge", use_lecam=True, perceptual_frames=4, lr_vae=1e-4, lr_disc=2e-4)
    out = tr.step(clip)        # clip: fp32 [B, 3, T, H, W] on cuda

Out of scope: DDP / NCCL (one process), CUDA-graph capture (the step runs eagerly), the latent flip and crop
augmentations, and HR decoding of the image Trainer.
"""
from __future__ import annotations

import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import torch
import torch.nn as nn
import torch.nn.functional as F

import tae
from flat import FlatAdamW
from vae_trainer import gan_disc_loss, gradnorm, vae_loss_function


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
    """Trainer._step_body (vae_trainer.py) on frames folded into the batch, in one process.

    vae: a float32 tae.TVAE; it is opted into training here (tae.enable_training; `recompute` passes through).
    lpips: utils.LPIPS (frozen; its train/eval mode is kept as given), or None for the MSE-only baseline, whose
        reconstruction term is F.mse_loss over the selected frames instead of the gradnormed LPIPS mean.
    discriminator: utils.PatchDiscriminator or None (no GAN terms). disc_type "hinge" or "bce"; use_lecam adds the
        LeCam regulariser with the anchors of Trainer (weight 0.1, EMA 0.9).
    perceptual_frames: k draws k distinct frames per clip per step from torch's CPU generator (torch.manual_seed makes
        runs reproducible); LPIPS, the MSE term and both GAN passes use that one selection. None: every frame.
    lr_vae, lr_disc: learning rates of the fused AdamW (vqb_adamw_flat; betas (0.9, 0.95), weight decay 1e-3, as in
        Trainer) over the TVAE and the discriminator.

    step(clip) per step:
      1. decz, z = vae(clip) (the reparameterisation draws its noise from torch's CUDA generator);
      2. with a discriminator: D on real and detached fake frames, hinge / BCE loss (+ LeCam), AdamW step of D;
      3. LPIPS(gradnorm(decz), clip).mean() over the selected frames, vae_loss_function(clip, gradnorm(decz, 0.001),
         z) with z the NCTHW encoder output (0.1 * mean(z^2)), and the generator loss of D on gradnorm(decz, 1.0) with
         D's parameters frozen for that pass; one backward, AdamW step of the TVAE.
    """

    def __init__(self, vae: nn.Module, lpips, discriminator=None, *, disc_type="hinge", use_lecam=False,
                 perceptual_frames=None, lr_vae, lr_disc=None, recompute=False):
        if disc_type not in ("hinge", "bce"):
            raise ValueError(f"unknown disc_type {disc_type!r}")
        if discriminator is not None and lr_disc is None:
            raise ValueError("lr_disc is required with a discriminator")
        if perceptual_frames is not None and perceptual_frames < 1:
            raise ValueError(f"perceptual_frames must be >= 1, got {perceptual_frames}")
        self.vae = tae.enable_training(vae, recompute=recompute)
        self.lpips, self.disc = lpips, discriminator
        self.disc_type, self.use_lecam, self.perceptual_frames = disc_type, use_lecam, perceptual_frames
        self.optimizer_G = FlatAdamW([{"params": [p for p in vae.parameters() if p.requires_grad], "lr": lr_vae}],
                                     weight_decay=1e-3, betas=(0.9, 0.95))
        self.optimizer_D = None
        device = next(vae.parameters()).device
        if discriminator is not None:
            discriminator.requires_grad_(True)
            self.optimizer_D = FlatAdamW([{"params": list(discriminator.parameters()), "lr": lr_disc}],
                                         weight_decay=1e-3, betas=(0.9, 0.95))
        self.lecam_loss_weight, self.lecam_beta = 0.1, 0.9
        self.lecam_anchor_real_logits = torch.zeros((), device=device)
        self.lecam_anchor_fake_logits = torch.zeros((), device=device)
        self.last_frames = None

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
        disc = self.disc
        decz, z = self.vae(clip)

        out = {}
        if disc is not None:
            real_preds = disc(clip, frames=sel)
            fake_preds = disc(decz.detach(), frames=sel)
            d_loss, avg_real_logits, avg_fake_logits, disc_acc = gan_disc_loss(real_preds, fake_preds, self.disc_type)
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
            self.optimizer_D.step()
            out.update(avg_real_logits=avg_real_logits, avg_fake_logits=avg_fake_logits, disc_acc=disc_acc,
                       lecam_loss=lecam_loss_item)

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

        self.optimizer_G.zero_grad(set_to_none=True)
        overall_vae_loss.backward()
        self.optimizer_G.step()
        out.update(overall_vae_loss=overall_vae_loss.detach(), perceptual_loss=recon_loss.detach(),
                   loss_data=loss_data, z=z.detach(), reconstructed=decz.detach())
        return out
