"""Per-frame image losses on [B, C, T, H, W] clips: the reference image modules applied to the selected frames folded
into the batch in (b, t) order, i.e. to rearrange(x[:, :, sel], "b c t h w -> (b t) c h w") with a per-clip selection.
The reference has no video trainer, so this is the definition of utils.LPIPS / utils.PatchDiscriminator on a clip and of
the losses of tae_trainer.VideoTrainer (DESIGN.md section 7). TEST INFRASTRUCTURE (see oracle/__init__.py).
"""
from __future__ import annotations

import torch

from oracle import lpips_oracle as LP


def fold_frames(x, frames=None):
    """[B, C, T, H, W] -> [B*T', C, H, W]: image b*T' + j is frame frames[b][j] of clip b (every frame when None)."""
    B, C, T, H, W = x.shape
    if frames is None:
        return x.transpose(1, 2).reshape(B * T, C, H, W)
    f = torch.as_tensor(frames, dtype=torch.long, device=x.device)
    idx = f.reshape(B, -1, 1, 1, 1).expand(B, f.shape[1], C, H, W)
    return torch.gather(x.transpose(1, 2), 1, idx).reshape(-1, C, H, W)


def lpips_clip(sd, inp, tgt, frames=None, keep_masks=None):
    """-> [B*T', 1, 1, 1] (keep_masks: the five train-mode dropout masks of the folded batch, as in lpips_forward)."""
    return LP.lpips_forward(sd, fold_frames(inp, frames), fold_frames(tgt, frames), keep_masks)


def patchd_clip(sd, x, frames=None):
    """-> [B*T', (H/16)(W/16)]."""
    return LP.patchd_forward(sd, fold_frames(x, frames))
