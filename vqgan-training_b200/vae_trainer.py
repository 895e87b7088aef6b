"""H100-native drop-in for the reference `vae_trainer.py` (the torchrun DDP entry, its CLI flags and the loss/autograd
glue): GradNormFunction / gradnorm / avg_scalar_over_nodes / gan_disc_loss / vae_loss_function / blurriness_heatmap /
create_dataloader / cleanup / train_ddp keep their names and argument meaning (vae_trainer.py:27-338); the step
ordering of the loop follows vae_trainer.py:524-710.

What differs from the reference, on purpose (DESIGN.md "Deviations"):
  * VAE gradients ARE all-reduced (the reference wraps the VAE in DDP but calls vae.module.* directly, so its reducer
    never fires — SURVEY.md fact 3). Gradients of VAE and discriminator are averaged with one flat NCCL all-reduce each.
  * no per-step host synchronisation: the ~15 `.item()` calls and the CPU z-statistics of the reference are evaluated
    only on logging steps; GradNorm's norm -> all-reduce -> rescale chain stays on the device.
  * the discriminator's wasted second backward (weight gradients thrown away at :706-708) is not executed.
  * `--dataset_url synthetic` (the default here) feeds seeded synthetic batches; webdataset is used when installed and a
    real URL is given (the reference overwrites the flag with the author's local path, :386-387).
  * `lecam_loss_item` is always defined (the reference NameErrors with --do_ganloss but without --use_lecam).
"""
from __future__ import annotations

import logging
import math
import os
import random
import sys
import time

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import click
import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F
import torch.optim as optim

from ae import VAE, enable_recompute
from utils import LPIPS, PatchDiscriminator, prepare_filter

try:  # optional: only needed for real datasets
    import webdataset as wds
except Exception:  # pragma: no cover
    wds = None
try:
    import wandb
except Exception:  # pragma: no cover
    wandb = None


def _dist_on():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


class GradNormFunction(torch.autograd.Function):
    """vae_trainer.py:27-48. Forward: clone. Backward: weight * g / (mean over ranks of ||g||_2 + 1e-8).
    The norm, its rank average and the rescale stay on the device (no .item())."""

    @staticmethod
    def forward(ctx, x, weight):
        # `weight` may be a python number (what gradnorm() passes: no host->device tensor creation inside the step, which
        # keeps the step CUDA-graph capturable) or a 0-dim tensor (the reference's calling convention, :51-53)
        ctx.weight = weight
        return x.clone()

    @staticmethod
    def backward(ctx, grad_output):
        weight = ctx.weight
        n = torch.linalg.vector_norm(grad_output.float())
        if _dist_on():
            dist.all_reduce(n, op=dist.ReduceOp.AVG)
        if torch.is_tensor(weight):
            weight = weight.to(device=grad_output.device, dtype=grad_output.dtype)
        return (weight / (n + 1e-8).to(grad_output.dtype)) * grad_output, None


def gradnorm(x, weight=1.0):
    return GradNormFunction.apply(x, weight)


@torch.no_grad()
def avg_scalar_over_nodes(value, device):
    """vae_trainer.py:56-60. Float in -> float out (host sync, reference behaviour); tensor in -> tensor out (no sync)."""
    if torch.is_tensor(value):
        v = value.detach().clone().float()
        if _dist_on():
            dist.all_reduce(v, op=dist.ReduceOp.AVG)
        return v
    v = torch.tensor(float(value), device=device)
    if _dist_on():
        dist.all_reduce(v, op=dist.ReduceOp.AVG)
    return v.item()


def gan_disc_loss(real_preds, fake_preds, disc_type="bce"):
    """vae_trainer.py:63-90 -> (loss, avg_real, avg_fake, acc). The three statistics are 0-dim device tensors
    (float() them to log) instead of python floats, so the training step never stalls the host."""
    if disc_type == "bce":
        real_loss = F.binary_cross_entropy_with_logits(real_preds, torch.ones_like(real_preds))
        fake_loss = F.binary_cross_entropy_with_logits(fake_preds, torch.zeros_like(fake_preds))
    elif disc_type == "hinge":
        real_loss = F.relu(1 - real_preds).mean()
        fake_loss = F.relu(1 + fake_preds).mean()
    else:
        raise ValueError(f"unknown disc_type {disc_type!r}")
    with torch.no_grad():
        acc = ((real_preds > 0).sum() + (fake_preds < 0).sum()).float() / (real_preds.numel() + fake_preds.numel())
        avg_real_preds = real_preds.mean()
        avg_fake_preds = fake_preds.mean()
    return (real_loss + fake_loss) * 0.5, avg_real_preds, avg_fake_preds, acc


MAX_WIDTH = 512


def create_dataloader(url, batch_size, num_workers, do_shuffle=True, just_resize=False):
    """vae_trainer.py:119-140 (webdataset) — or a synthetic stream when url == 'synthetic' / webdataset is missing."""
    if url in ("", "synthetic") or wds is None:
        return SyntheticLoader(batch_size, MAX_WIDTH)
    import torchvision.transforms as transforms

    def rc(x, width=MAX_WIDTH):  # this_transform_random_crop_resize, vae_trainer.py:105-116
        x = transforms.ToTensor()(x)
        x = transforms.Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5])(x)
        if random.random() < 0.5:
            return transforms.RandomCrop(width)(x)
        return transforms.RandomCrop(width)(transforms.Resize(width)(x))

    plain = transforms.Compose([transforms.ToTensor(), transforms.Normalize([0.5] * 3, [0.5] * 3),
                                transforms.CenterCrop(512), transforms.Resize(MAX_WIDTH)])
    dataset = wds.WebDataset(url, nodesplitter=wds.split_by_node, workersplitter=wds.split_by_worker)
    dataset = dataset.shuffle(1000) if do_shuffle else dataset
    dataset = dataset.decode("rgb").to_tuple("jpg;png").map_tuple(rc if not just_resize else plain)
    return wds.WebLoader(dataset, batch_size=batch_size, shuffle=False, num_workers=num_workers, pin_memory=True)


class SyntheticLoader:
    """Endless seeded stream of pinned host batches in [-1, 1) (the range of Normalize(.5,.5), vae_trainer.py:98):
    images [B, 3, R, R], or clips [B, 3, frames, R, R] for the video trainer (tae_trainer.py)."""

    def __init__(self, batch_size, resolution, seed=None, n_distinct=4, frames=None):
        rank = int(os.environ.get("RANK", "0"))
        g = torch.Generator().manual_seed(42 + rank if seed is None else seed)
        shape = (batch_size, 3) + (() if frames is None else (frames,)) + (resolution, resolution)
        self.batches = [(torch.rand(shape, generator=g) * 2 - 1) for _ in range(n_distinct)]
        if torch.cuda.is_available():
            self.batches = [b.pin_memory() for b in self.batches]

    def __iter__(self):
        i = 0
        while True:
            yield (self.batches[i % len(self.batches)],)
            i += 1


def blurriness_heatmap(input_image):
    """vae_trainer.py:143-176 (5x5 Laplacian-like conv, |.|, 13x13 sigma-2 Gaussian with reflect padding, min/max
    normalisation over the whole batch tensor, threshold 0.8). Zero-weighted at HEAD; small 1-channel ATen ops."""
    gray = input_image.mean(dim=1, keepdim=True)
    lap = torch.tensor([[0, 1, 1, 1, 0], [1, 1, 1, 1, 1], [1, 1, -20, 1, 1], [1, 1, 1, 1, 1], [0, 1, 1, 1, 0]],
                       dtype=torch.float32, device=input_image.device).view(1, 1, 5, 5)
    edge = F.conv2d(gray, lap, padding=2).abs()
    half = 6.0
    xs = torch.linspace(-half, half, steps=13, device=input_image.device)
    k1 = torch.exp(-0.5 * (xs / 2.0).pow(2))
    k1 = k1 / k1.sum()
    edge = F.conv2d(F.pad(edge, (6, 6, 6, 6), mode="reflect"), (k1[:, None] * k1[None, :]).view(1, 1, 13, 13))
    edge = (edge - edge.min()) / (edge.max() - edge.min() + 1e-8)
    blur = 1 - edge
    blur = torch.where(blur < 0.8, torch.zeros_like(blur), blur)
    return blur.repeat(1, 3, 1, 1)


RECON_LOSS_WEIGHT = 0.0  # the literal `recon_loss * 0.0` of vae_trainer.py:209


def vae_loss_function(x, x_reconstructed, z, do_pool=True, do_recon=False):
    """vae_trainer.py:179-217 -> (loss, stats). stats hold 0-dim device tensors (float() to log)."""
    if do_recon:
        if do_pool:
            xr = F.interpolate(x_reconstructed, scale_factor=1 / 16, mode="area")
            xd = F.interpolate(x, scale_factor=1 / 16, mode="area")
            recon_loss = (xr - xd).abs().mean()
        else:
            recon_loss = ((x_reconstructed - x) * blurriness_heatmap(x)).abs().mean()
        recon_loss_item = recon_loss.detach()
    else:
        recon_loss = 0
        recon_loss_item = torch.zeros((), device=z.device)
    zloss = z.pow(2).mean()
    vae_loss = recon_loss * RECON_LOSS_WEIGHT + zloss * 0.1
    with torch.no_grad():
        az = z.abs()
        stats = {"recon_loss": recon_loss_item, "kl_loss": zloss.detach(), "average_of_abs_z": az.mean(),
                 "std_of_abs_z": az.std(), "average_of_logvar": 0.0, "std_of_logvar": 0.0}
    return vae_loss, stats


def cleanup():
    if dist.is_initialized():
        dist.destroy_process_group()


class FlatAllReduceDDP(nn.Module):
    """Data-parallel wrapper with the DDP surface the reference uses (`.module`, `module.`-prefixed state_dict,
    constructor broadcast from rank 0) whose gradient averaging is explicit — it therefore also covers the
    `vae.module.encoder(...)` calling style that bypasses DDP.forward in the reference (SURVEY.md fact 3).

    With a flat gradient store attached (`attach_store`, flat.FlatParams — what Trainer does) the weight-gradient kernels
    have already written into one contiguous fp32 buffer, so `allreduce_grads()` is ONE in-place NCCL all-reduce(AVG)
    with no copy-in / copy-out. VQB_DDP_OVERLAP=k (k >= 2, opt-in) splits that buffer into k contiguous ranges (in
    parameter registration order: the decoder's range completes first in backward) and launches each range's
    all-reduce asynchronously from a post-accumulate-grad hook as soon as its last gradient has landed;
    `allreduce_grads()` then only waits. Without a store (plain modules, tests) gradients are staged through a
    temporary flat buffer."""

    def __init__(self, module: nn.Module, device_ids=None):
        super().__init__()
        self.module = module
        if _dist_on():
            for t in list(module.parameters()) + list(module.buffers()):
                dist.broadcast(t.data, 0)
            if any(p.is_cuda for p in module.parameters()):
                import ops

                ops.weights_updated(list(module.parameters()))  # .data writes do not bump Tensor._version
        self._flat = None
        self._store = None
        self._ranges = None
        self.after_load = None  # load_vae_checkpoint calls this after the weights changed (a trainer's EMA restart)

    def forward(self, *a, **k):
        return self.module(*a, **k)

    def attach_store(self, store, overlap_ranges=None):
        """Gradients of this module live in `store.grads` (flat.FlatParams): all-reduce that buffer in place."""
        self._store = store
        k = int(os.environ.get("VQB_DDP_OVERLAP", "0")) if overlap_ranges is None else overlap_ranges
        if k >= 2 and _dist_on():
            self._build_ranges(k)

    def _build_ranges(self, k: int):
        st = self._store
        target = st.total / k
        self._ranges, self._range_of = [], {}
        lo = 0
        for r in range(k):
            hi = lo
            while hi < len(st.plist) and (r == k - 1 or st.offsets[hi] < target * (r + 1)):
                hi += 1
            if hi == lo:
                continue
            a = st.offsets[lo]
            b = st.offsets[hi] if hi < len(st.plist) else st.total
            self._ranges.append({"idx": range(lo, hi), "a": a, "b": b, "ready": 0, "work": None})
            lo = hi
        for ri, rg in enumerate(self._ranges):
            for i in rg["idx"]:
                p = st.plist[i]
                self._range_of[p] = ri
                p.register_post_accumulate_grad_hook(self._grad_ready)

    @torch.no_grad()
    def _launch_range(self, rg):
        st = self._store
        st.collect(rg["idx"])
        rg["work"] = dist.all_reduce(st.grads[rg["a"]:rg["b"]], op=dist.ReduceOp.AVG, async_op=True)

    @torch.no_grad()
    def _grad_ready(self, p):
        rg = self._ranges[self._range_of[p]]
        if rg["work"] is not None:
            raise RuntimeError("FlatAllReduceDDP: a second backward reached a range that is already being reduced; "
                               "call allreduce_grads() after every backward or unset VQB_DDP_OVERLAP")
        rg["ready"] += 1
        if rg["ready"] == len(rg["idx"]):
            self._launch_range(rg)

    @torch.no_grad()
    def allreduce_grads(self):
        if not _dist_on():
            return
        if self._store is not None:
            if self._ranges is None:
                self._store.collect()
                dist.all_reduce(self._store.grads, op=dist.ReduceOp.AVG)
                return
            for rg in self._ranges:
                if rg["work"] is None:  # some parameter of the range got no gradient this step (same on every rank)
                    self._launch_range(rg)
            for rg in self._ranges:
                rg["work"].wait()
                rg["work"], rg["ready"] = None, 0
            return
        params = [p for p in self.module.parameters() if p.requires_grad and p.grad is not None]
        if not params:
            return
        n = sum(p.numel() for p in params)
        if self._flat is None or self._flat.numel() != n:
            self._flat = torch.empty(n, device=params[0].device, dtype=torch.float32)
        off = 0
        views = []
        for p in params:
            v = self._flat[off:off + p.numel()].view_as(p)
            views.append(v)
            off += p.numel()
        torch._foreach_copy_(views, [p.grad for p in params])
        dist.all_reduce(self._flat, op=dist.ReduceOp.AVG)
        torch._foreach_copy_([p.grad for p in params], views)


def cosine_with_warmup(optimizer, num_warmup_steps, num_training_steps):
    """transformers.get_cosine_schedule_with_warmup (vae_trainer.py:486-490) without the dependency."""

    def f(step):
        if step < num_warmup_steps:
            return float(step) / float(max(1, num_warmup_steps))
        progress = float(step - num_warmup_steps) / float(max(1, num_training_steps - num_warmup_steps))
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * 2.0 * 0.5 * progress)))

    return optim.lr_scheduler.LambdaLR(optimizer, f)


def latent_augment(z, z_s, real_images_hr, flip_invariance, crop_invariance, downscale_factor=16,
                   decoder_also_perform_hr=False):
    """vae_trainer.py:567-621, the equivariance augmentations between encoder and decoder. Draw order of python's
    `random` is the reference's (three `random.random()` draws always happen; the crop's four `randint`s only when it
    fires):
      * horizontal flip of the latent with channels [-4:-2] negated + the same flip of the target image,
      * vertical flip with channels [-2:] negated,
      * a random crop of the latent (>= 12 latent pixels per side) and the matching crop of the target image.
    -> (z_s, real_images_hr)."""
    if random.random() < 0.5 and flip_invariance:  # :567-570
        z_s = torch.flip(z_s, [-1]).clone()
        z_s[:, -4:-2] = -z_s[:, -4:-2]
        real_images_hr = torch.flip(real_images_hr, [-1])
    if random.random() < 0.5 and flip_invariance:  # :572-575
        z_s = torch.flip(z_s, [-2]).clone()
        z_s[:, -2:] = -z_s[:, -2:]
        real_images_hr = torch.flip(real_images_hr, [-2])
    if random.random() < 0.5 and crop_invariance:  # :577-621
        z_h, z_w = z.shape[-2:]
        new_z_h, new_z_w = random.randint(12, z_h - 1), random.randint(12, z_w - 1)
        offset_z_h, offset_z_w = random.randint(0, z_h - new_z_h - 1), random.randint(0, z_w - new_z_w - 1)
        f = downscale_factor * (2 if decoder_also_perform_hr else 1)
        real_images_hr = real_images_hr[:, :, offset_z_h * f:(offset_z_h + new_z_h) * f,
                                        offset_z_w * f:(offset_z_w + new_z_w) * f]
        z_s = z_s[:, :, offset_z_h:offset_z_h + new_z_h, offset_z_w:offset_z_w + new_z_w]
        assert real_images_hr.shape[-2:] == (new_z_h * f, new_z_w * f) and z_s.shape[-2:] == (new_z_h, new_z_w)
    return z_s, real_images_hr


def load_vae_checkpoint(vae_ddp: nn.Module, path_or_state):
    """vae_trainer.py:505-513: strict load of a `module.`-prefixed VAE checkpoint (what the reference saves at :903-906);
    on failure the `_orig_mod.` infixes a torch.compile'd encoder/decoder leaves in the keys are stripped and the strict
    load is retried. After loading, the cached bf16 GEMM operands are refreshed and, when the wrapper belongs to a
    trainer that keeps a weight EMA, that average restarts from the loaded weights."""
    state_dict = torch.load(path_or_state, map_location="cpu") if isinstance(path_or_state, (str, os.PathLike)) \
        else path_or_state
    try:
        status = vae_ddp.load_state_dict(state_dict, strict=True)
    except Exception as e:
        print(e)
        state_dict = {k.replace("_orig_mod.", ""): v for k, v in state_dict.items()}
        status = vae_ddp.load_state_dict(state_dict, strict=True)
        print(status)
    if any(p.is_cuda for p in vae_ddp.parameters()):
        import ops

        ops.weights_updated(list(vae_ddp.parameters()))
    if getattr(vae_ddp, "after_load", None) is not None:
        vae_ddp.after_load()
    return status


def make_image_grid(images: torch.Tensor, D: int) -> torch.Tensor:
    """vae_trainer.py:872-893: the first 8 images, cropped to D x D, tiled 2 rows x 4 columns into a (3, 4D, 4D) canvas
    (the reference allocates 4D x 4D and fills the top half)."""
    canvas = torch.zeros((3, D * 4, D * 4))
    images = images[:, :, :D, :D].cpu()
    for i in range(2):
        for j in range(4):
            if i * 4 + j < images.shape[0]:
                img = images[i * 4 + j]
                canvas[:, i * D:i * D + img.shape[-2], j * D:j * D + img.shape[-1]] = img
    return canvas


@torch.no_grad()
def restart_ema(optimizer, live: nn.Module, averaged: nn.Module):
    """Restarts `optimizer`'s weight EMA from the current weights of `live` and copies `live`'s frozen parameters and
    buffers into `averaged` (its FlatAdamW.averaged_copy)."""
    optimizer.reset_ema()
    trained = {id(p) for p in optimizer.store.plist}
    for a, b in zip(averaged.parameters(), live.parameters()):
        if id(b) not in trained:
            a.copy_(b)
    for a, b in zip(averaged.buffers(), live.buffers()):
        a.copy_(b)


class Trainer:
    """One object = the state of vae_trainer.py:422-522 (models, optimizers, scheduler, LeCam anchors); `.step(batch)`
    = one iteration of the loop body :530-708. bench.py and the tests drive this same public class."""

    def __init__(self, device, vae_resolution=256, vae_in_channels=3, vae_ch=256, vae_ch_mult="1,2,4,4",
                 vae_num_res_blocks=2, vae_z_channels=16, do_attn=False, decoder_also_perform_hr=False,
                 use_wavelet=False, do_ganloss=False, learning_rate_vae=1e-5, learning_rate_disc=2e-4, max_steps=1000,
                 do_clamp=False, clamp_th=8.0, crop_invariance=False, flip_invariance=False,
                 augment_before_perceptual_loss=False, downscale_factor=16, use_lecam=False, disc_type="bce",
                 lpips_eval=True, seed=42, use_vq=False, vq_codebook_size=8192, vq_beta=0.25, cuda_graph=None,
                 recompute=False, ema_decay=None):
        """recompute=True: ae.enable_recompute on the VAE, so that every ResnetBlock keeps only its input for the
        backward (larger batches or resolutions per GPU for one extra conv1 and two GroupNorm apply passes per block).
        ema_decay (0 < d < 1): keep an exponential moving average of the VAE's weights (every parameter of optimizer_G,
        the VQ codebook included) in the fused AdamW launch (flat.FlatAdamW); `vae_ema` is an ae.VAE over it. None: no
        average (vae_ema is None)."""
        if ema_decay is not None:
            from flat import check_ema_decay

            ema_decay = check_ema_decay(ema_decay)  # before any device work
        self.device = device
        # CUDA-graph the whole step (forward, backward, NCCL collectives, optimizers, weight re-pack): ~600-1100 launches
        # per step otherwise keep the host within ~10 % of being the limiter. Auto-enabled (None) when no host-side
        # random branch changes the graph from step to step; VQB_CUDA_GRAPH=0 disables.
        if cuda_graph is None:
            # multi-rank: the captured step contains the NCCL collectives (N=2: 665.7 vs 659.6 images/s eager-launched;
            # release_graph() before destroy_process_group()). VQB_CUDA_GRAPH=0 disables, =single keeps it to one rank.
            mode = os.environ.get("VQB_CUDA_GRAPH", "1")
            cuda_graph = mode == "1" or (mode == "single" and not _dist_on())
        # (LPIPS in train mode draws fresh dropout seeds on the host every call: a replayed graph would freeze the mask,
        # so the train-mode metric — what train_ddp uses, like the reference — runs the eager-launched step)
        self._graph_wanted = bool(cuda_graph) and lpips_eval and not (crop_invariance or flip_invariance or
                                                                      augment_before_perceptual_loss)
        self._graph = None          # (key, CUDAGraph, static input, static outputs, launches per step)
        self._graph_warm = 0
        self.do_ganloss, self.do_clamp, self.clamp_th = do_ganloss, do_clamp, clamp_th
        self.crop_invariance, self.flip_invariance = crop_invariance, flip_invariance
        self.augment_before_perceptual_loss = augment_before_perceptual_loss
        self.downscale_factor, self.use_lecam, self.disc_type = downscale_factor, use_lecam, disc_type
        self.decoder_also_perform_hr = decoder_also_perform_hr

        torch.manual_seed(seed)           # vae_trainer.py:374-378
        torch.cuda.manual_seed_all(seed)
        np.random.seed(seed)
        random.seed(seed)

        vae = VAE(resolution=vae_resolution, in_channels=vae_in_channels, ch=vae_ch, out_ch=vae_in_channels,
                  ch_mult=[int(x) for x in str(vae_ch_mult).split(",")], num_res_blocks=vae_num_res_blocks,
                  z_channels=vae_z_channels, use_attn=do_attn, decoder_also_perform_hr=decoder_also_perform_hr,
                  use_wavelet=use_wavelet).to(device)
        if recompute:
            enable_recompute(vae)
        self.use_vq = use_vq
        if use_vq:  # BASELINE.json config 4: the codebook replaces vae.module.reg (vae_trainer.py:563)
            from ae import VectorQuantizer

            vae.reg = VectorQuantizer(vq_codebook_size, vae_z_channels, vq_beta).to(device)
        discriminator = PatchDiscriminator().to(device)
        discriminator.requires_grad_(True)
        self.vae = FlatAllReduceDDP(vae)
        prepare_filter(device)
        self.discriminator = FlatAllReduceDDP(discriminator)

        # vae_trainer.py:455-475: two AdamW groups for the VAE (conv_in at 1e-4, the rest at lr/ch), one for D — as ONE
        # fused kernel each over flat parameter/gradient/moment buffers (flat.FlatAdamW). The [extension] VQ codebook
        # gets its own group at the un-divided VAE learning rate (it would never move at lr/ch).
        from flat import FlatAdamW

        named = list(self.vae.named_parameters())
        groups = [{"params": [p for n, p in named if "conv_in" not in n and "reg.embedding" not in n],
                   "lr": learning_rate_vae / vae_ch},
                  {"params": [p for n, p in named if "conv_in" in n], "lr": 1e-4}]
        if use_vq:
            groups.append({"params": [p for n, p in named if "reg.embedding" in n], "lr": learning_rate_vae})
        self.optimizer_G = FlatAdamW(groups, weight_decay=1e-3, betas=(0.9, 0.95), ema_decay=ema_decay)
        self.optimizer_D = FlatAdamW([{"params": list(self.discriminator.parameters()), "lr": learning_rate_disc}],
                                     weight_decay=1e-3, betas=(0.9, 0.95))
        self.vae.attach_store(self.optimizer_G.store)
        self.discriminator.attach_store(self.optimizer_D.store)
        # [extension] the weight EMA (DESIGN.md section 7 row 26): the autoencoder only, started after the broadcast above
        self.vae_ema = None
        if ema_decay is not None:
            self.vae_ema = self.optimizer_G.averaged_copy(vae)
            self.vae.after_load = lambda: restart_ema(self.optimizer_G, self.vae.module, self.vae_ema)
        self.lpips = LPIPS().to(device)
        from utils import broadcast_module_state

        broadcast_module_state(self.lpips)  # frozen, not DDP-wrapped: every rank must score with rank 0's weights
        if lpips_eval:
            self.lpips.eval()
        self.lr_scheduler = cosine_with_warmup(self.optimizer_G, 200, max_steps)
        self.lecam_loss_weight, self.lecam_beta = 0.1, 0.9
        self.lecam_anchor_real_logits = torch.zeros((), device=device)
        self.lecam_anchor_fake_logits = torch.zeros((), device=device)
        self.global_step = 0
        self.last = {}

    GRAPH_WARMUP_STEPS = 3

    def step(self, real_images_hr: torch.Tensor):
        """One iteration of vae_trainer.py:530-708. Host-side random decisions (the horizontal flip of :534-536 and the
        draws of the equivariance augmentations) are taken here, in the reference's order; the device work runs either
        eagerly or — after GRAPH_WARMUP_STEPS eager steps — as one CUDA-graph replay."""
        flip = random.random() < 0.5  # :534-536
        key = (tuple(real_images_hr.shape), real_images_hr.dtype)
        use_graph = self._graph_wanted and real_images_hr.dtype == torch.float32 and \
            (self._graph is None or self._graph[0] == key)
        if not use_graph or self._graph_warm < self.GRAPH_WARMUP_STEPS:
            self._graph_warm += 1
            x = real_images_hr.to(self.device, non_blocking=True)
            if flip:
                x = torch.flip(x, [-1])
            out = self._step_body(x, graph_mode=False)
        else:
            out = self._step_graph(real_images_hr, flip, key)
            for _ in range(3):
                random.random()  # the three draws of latent_augment (:567,572,577), which the replay does not execute
        self.lr_scheduler.step()
        self.global_step += 1
        self.last = out
        return out

    def _step_graph(self, real_images_hr, flip, key):
        if self._graph is None:
            static_in = torch.empty(key[0], device=self.device, dtype=torch.float32)
            static_in.copy_(real_images_hr, non_blocking=True)
            import native

            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            st_state = random.getstate()
            l0 = native.launch_count()
            with torch.cuda.graph(g):
                out = self._step_body(static_in, graph_mode=True)
            random.setstate(st_state)  # the capture ran the python body once: its draws are re-done by step()
            self._graph = (key, g, static_in, out, native.launch_count() - l0)
        _, g, static_in, out, _ = self._graph
        if flip:
            static_in.copy_(torch.flip(real_images_hr.to(self.device, non_blocking=True), [-1]))
        else:
            static_in.copy_(real_images_hr, non_blocking=True)
        self.optimizer_G.upload_hyper()
        if self.do_ganloss:
            self.optimizer_D.upload_hyper()
        g.replay()
        return out

    def release_graph(self):
        """Drops the captured step (and the memory pool it pins). Call before destroying the process group."""
        self._graph = None
        self._graph_wanted = False
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    @property
    def graph_launches_per_step(self):
        """Kernels of libvqb200.so inside one replay of the captured step (None while running eagerly)."""
        return self._graph[4] if self._graph is not None else None

    def _opt_step(self, opt, graph_mode):
        if graph_mode:  # capturable form: the hyper-parameter record is uploaded by _step_graph before every replay
            active = opt.store.collect()
            opt.launch(active, pack=True)
        else:
            opt.step()

    def _step_body(self, real_images_hr: torch.Tensor, graph_mode: bool):
        vae, disc = self.vae, self.discriminator
        device = self.device
        if real_images_hr.shape[-2:] != (256, 256):
            real_images_for_enc = F.interpolate(real_images_hr, size=(256, 256), mode="area")  # :531-533
        else:
            real_images_for_enc = real_images_hr  # the area resize is an exact identity at 256^2

        z = vae.module.encoder(real_images_for_enc)  # :538
        z_for_stats = z.detach()
        if self.do_clamp:
            z = z.clamp(-self.clamp_th, self.clamp_th)
        vq_loss = None
        if self.use_vq:
            z_s, vq_loss, _ = vae.module.reg(z)
        else:
            z_s = vae.module.reg(z)

        z_s, real_images_hr = latent_augment(z, z_s, real_images_hr, self.flip_invariance, self.crop_invariance,
                                             self.downscale_factor, self.decoder_also_perform_hr)  # :567-621
        real_images_hr = real_images_hr.contiguous()

        reconstructed = vae.module.decoder(z_s.contiguous())  # :623-624

        out = {}
        if self.do_ganloss:  # :629-659
            real_preds = disc(real_images_hr)
            fake_preds = disc(reconstructed.detach())
            d_loss, avg_real_logits, avg_fake_logits, disc_acc = gan_disc_loss(real_preds, fake_preds, self.disc_type)
            avg_real_logits = avg_scalar_over_nodes(avg_real_logits, device)
            avg_fake_logits = avg_scalar_over_nodes(avg_fake_logits, device)
            # in place: the anchors are persistent device scalars (also across CUDA-graph replays)
            self.lecam_anchor_real_logits.mul_(self.lecam_beta).add_(avg_real_logits, alpha=1 - self.lecam_beta)
            self.lecam_anchor_fake_logits.mul_(self.lecam_beta).add_(avg_fake_logits, alpha=1 - self.lecam_beta)
            total_d_loss = d_loss.mean()
            out["d_loss"] = total_d_loss.detach()
            lecam_loss_item = torch.zeros((), device=device)
            if self.use_lecam:
                lecam_loss = (real_preds - self.lecam_anchor_fake_logits).pow(2).mean() + \
                    (fake_preds - self.lecam_anchor_real_logits).pow(2).mean()
                lecam_loss_item = lecam_loss.detach()
                total_d_loss = total_d_loss + lecam_loss * self.lecam_loss_weight
            self.optimizer_D.zero_grad(set_to_none=True)
            total_d_loss.backward()
            disc.allreduce_grads()
            self._opt_step(self.optimizer_D, graph_mode)
            out.update(avg_real_logits=avg_real_logits, avg_fake_logits=avg_fake_logits, disc_acc=disc_acc,
                       lecam_loss=lecam_loss_item)

        _recon_for_perceptual = gradnorm(reconstructed)  # :662
        if self.augment_before_perceptual_loss:  # :664-674
            real_images_hr_aug = real_images_hr.clone()
            if random.random() < 0.5:
                _recon_for_perceptual = torch.flip(_recon_for_perceptual, [-1])
                real_images_hr_aug = torch.flip(real_images_hr_aug, [-1])
            if random.random() < 0.5:
                _recon_for_perceptual = torch.flip(_recon_for_perceptual, [-2])
                real_images_hr_aug = torch.flip(real_images_hr_aug, [-2])
        else:
            real_images_hr_aug = real_images_hr
        percep_rec_loss = self.lpips(_recon_for_perceptual, real_images_hr_aug).mean()  # :676

        recon_for_mse = gradnorm(reconstructed, weight=0.001)  # :679
        vae_loss, loss_data = vae_loss_function(real_images_hr, recon_for_mse, z)  # :680
        if self.do_ganloss:  # :682-696
            recon_for_gan = gradnorm(reconstructed, weight=1.0)
            disc.module.requires_grad_(False)  # the G pass needs D's data gradient only (no wasted wgrad/all-reduce)
            fake_preds = disc(recon_for_gan)
            disc.module.requires_grad_(True)
            if self.disc_type == "bce":
                g_gan_loss = F.binary_cross_entropy_with_logits(fake_preds, torch.ones_like(fake_preds))
            else:
                g_gan_loss = -fake_preds.mean()
            overall_vae_loss = percep_rec_loss + g_gan_loss + vae_loss
            out["g_gan_loss"] = g_gan_loss.detach()
        else:
            overall_vae_loss = percep_rec_loss + vae_loss
        if vq_loss is not None:
            overall_vae_loss = overall_vae_loss + vq_loss
            out["vq_loss"] = vq_loss.detach()

        overall_vae_loss.backward()  # :701
        vae.allreduce_grads()        # the all-reduce the reference intends (SURVEY.md fact 3)
        self._opt_step(self.optimizer_G, graph_mode)
        self.optimizer_G.zero_grad(set_to_none=True)
        out.update(overall_vae_loss=overall_vae_loss.detach(), perceptual_loss=percep_rec_loss.detach(),
                   loss_data=loss_data, z=z_for_stats, reconstructed=reconstructed.detach())
        return out

    @torch.no_grad()
    def evaluate(self, test_batches, max_batches=2, ema=False):
        """vae_trainer.py:811-893 (rank 0): encode the 256^2 area-resized test images, clamp, reg, [flip_invariance: decode
        the (-1,-2)-flipped latent with its last four channels negated and flip the image back, :837-861], decode,
        un-normalise to [0,1]. -> (test grid, reconstruction grid) as (3, 4D, 4D) tensors + the raw tensors.
        ema=True reconstructs with the averaged weights (vae_ema) instead of the trained ones."""
        if ema and self.vae_ema is None:
            raise ValueError("evaluate(ema=True): this trainer keeps no weight EMA (ema_decay=None)")
        model = self.vae_ema if ema else self.vae.module
        all_test, all_rec = [], []
        for batch in test_batches:
            ori = (batch[0] if isinstance(batch, (tuple, list)) else batch).to(self.device)
            x = F.interpolate(ori, size=(256, 256), mode="area") if ori.shape[-2:] != (256, 256) else ori
            z = model.encoder(x)
            if self.do_clamp:
                z = z.clamp(-self.clamp_th, self.clamp_th)
            z_s = model.reg(z)
            if isinstance(z_s, tuple):
                z_s = z_s[0]
            if self.flip_invariance:
                z_s = torch.flip(z_s, [-1, -2]).clone()
                z_s[:, -4:] = -z_s[:, -4:]
            rec = model.decoder(z_s.contiguous())
            ori, rec = (ori * 0.5 + 0.5).clamp(0, 1), (rec * 0.5 + 0.5).clamp(0, 1)
            if self.flip_invariance:
                rec = torch.flip(rec, [-1, -2])
            all_test.append(ori)
            all_rec.append(rec)
            if len(all_test) >= max_batches:
                break
        test_images, reconstructed = torch.cat(all_test, 0), torch.cat(all_rec, 0)
        D = 512 if self.decoder_also_perform_hr else 256
        return {"test_images": make_image_grid(test_images, D), "reconstructed_test_images":
                make_image_grid(reconstructed, D), "raw_test": test_images, "raw_reconstructed": reconstructed}

    def z_quantiles(self, z):
        """vae_trainer.py:541-559, evaluated only when something is logged."""
        v = z.float().reshape(-1).cpu()
        if v.numel() > 2 ** 24:
            v = v[:: v.numel() // 2 ** 24 + 1]
        kurt = ((v - v.mean()) ** 4).mean() / (v.std() ** 4)
        skew = ((v - v.mean()) ** 3).mean() / (v.std() ** 3)
        q = {f"{p:.1f}": v.quantile(p) for p in (0.0, 0.2, 0.4, 0.6, 0.8, 1.0)}
        q.update(kurtosis=kurt, skewness=skew)
        return q


@click.command()
@click.option("--dataset_url", type=str, default="synthetic", help="URL for the training dataset ('synthetic' = seeded random batches)")
@click.option("--test_dataset_url", type=str, default="synthetic", help="URL for the test dataset")
@click.option("--num_epochs", type=int, default=2, help="Number of training epochs")
@click.option("--batch_size", type=int, default=8, help="Batch size for training")
@click.option("--do_ganloss", is_flag=True, help="Whether to use GAN loss")
@click.option("--learning_rate_vae", type=float, default=1e-5, help="Learning rate for VAE")
@click.option("--learning_rate_disc", type=float, default=2e-4, help="Learning rate for discriminator")
@click.option("--vae_resolution", type=int, default=256, help="Resolution for VAE")
@click.option("--vae_in_channels", type=int, default=3, help="Input channels for VAE")
@click.option("--vae_ch", type=int, default=256, help="Base channel size for VAE")
@click.option("--vae_ch_mult", type=str, default="1,2,4,4", help="Channel multipliers for VAE")
@click.option("--vae_num_res_blocks", type=int, default=2, help="Number of residual blocks for VAE")
@click.option("--vae_z_channels", type=int, default=16, help="Number of latent channels for VAE")
@click.option("--run_name", type=str, default="run", help="Name of the run for wandb")
@click.option("--max_steps", type=int, default=1000, help="Maximum number of steps to train for")
@click.option("--evaluate_every_n_steps", type=int, default=250, help="Evaluate every n steps")
@click.option("--load_path", type=str, default=None, help="Path to load the model from")
@click.option("--do_clamp", is_flag=True, help="Whether to clamp the latent codes")
@click.option("--clamp_th", type=float, default=8.0, help="Clamp threshold for the latent codes")
@click.option("--max_spatial_dim", type=int, default=256, help="Maximum spatial dimension for overall training")
@click.option("--do_attn", type=bool, default=False, help="Whether to use attention in the VAE")
@click.option("--decoder_also_perform_hr", type=bool, default=False, help="Whether to perform HR decoding in the decoder")
@click.option("--project_name", type=str, default="vae_sweep_attn_lr_width", help="Project name for wandb")
@click.option("--crop_invariance", type=bool, default=False, help="Whether to perform crop invariance")
@click.option("--flip_invariance", type=bool, default=False, help="Whether to perform flip invariance")
@click.option("--do_compile", type=bool, default=False, help="Accepted for CLI compatibility; ignored (no tracing compiler on this path)")
@click.option("--use_wavelet", type=bool, default=False, help="Whether to use wavelet transform in the encoder")
@click.option("--augment_before_perceptual_loss", type=bool, default=False, help="Whether to augment the images before the perceptual loss")
@click.option("--downscale_factor", type=int, default=16, help="Downscale factor for the latent space")
@click.option("--use_lecam", type=bool, default=False, help="Whether to use Lecam")
@click.option("--disc_type", type=str, default="bce", help="Discriminator type")
@click.option("--use_vq", type=bool, default=False, help="[extension] VQ codebook bottleneck instead of reg (BASELINE config 4)")
@click.option("--vq_codebook_size", type=int, default=8192, help="[extension] number of codebook entries")
@click.option("--vq_beta", type=float, default=0.25, help="[extension] commitment loss weight")
def train_ddp(dataset_url, test_dataset_url, num_epochs, batch_size, do_ganloss, learning_rate_vae, learning_rate_disc,
              vae_resolution, vae_in_channels, vae_ch, vae_ch_mult, vae_num_res_blocks, vae_z_channels, run_name,
              max_steps, evaluate_every_n_steps, load_path, do_clamp, clamp_th, max_spatial_dim, do_attn,
              decoder_also_perform_hr, project_name, crop_invariance, flip_invariance, do_compile, use_wavelet,
              augment_before_perceptual_loss, downscale_factor, use_lecam, disc_type, use_vq, vq_codebook_size, vq_beta):
    assert torch.cuda.is_available(), "CUDA is required for DDP"
    ddp_rank = int(os.environ.get("RANK", "0"))
    ddp_local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world_size = int(os.environ.get("WORLD_SIZE", "1"))
    device = f"cuda:{ddp_local_rank}"
    torch.cuda.set_device(device)
    if "RANK" in os.environ:
        dist.init_process_group(backend="nccl", device_id=torch.device(device))
    master_process = ddp_rank == 0
    print(f"using device: {device}")

    use_wandb = master_process and wandb is not None and os.environ.get("WANDB_MODE", "") != "disabled" \
        and os.environ.get("VQB_WANDB", "0") == "1"
    if use_wandb:
        wandb.init(project=project_name, name=run_name, config=dict(
            learning_rate_vae=learning_rate_vae, learning_rate_disc=learning_rate_disc, vae_ch=vae_ch,
            vae_resolution=vae_resolution, vae_in_channels=vae_in_channels, vae_ch_mult=vae_ch_mult,
            vae_num_res_blocks=vae_num_res_blocks, vae_z_channels=vae_z_channels, batch_size=batch_size,
            num_epochs=num_epochs, do_ganloss=do_ganloss, do_attn=do_attn, use_wavelet=use_wavelet))

    tr = Trainer(device, vae_resolution, vae_in_channels, vae_ch, vae_ch_mult, vae_num_res_blocks, vae_z_channels,
                 do_attn, decoder_also_perform_hr, use_wavelet, do_ganloss, learning_rate_vae, learning_rate_disc,
                 max_steps, do_clamp, clamp_th, crop_invariance, flip_invariance, augment_before_perceptual_loss,
                 downscale_factor, use_lecam, disc_type, lpips_eval=False, use_vq=use_vq,
                 vq_codebook_size=vq_codebook_size, vq_beta=vq_beta)

    logger = logging.getLogger(__name__)
    logger.setLevel(logging.INFO)
    if master_process:
        handler = logging.StreamHandler()
        handler.setFormatter(logging.Formatter("%(asctime)s - %(name)s - %(levelname)s - %(message)s"))
        logger.addHandler(handler)

    if load_path is not None:  # :505-513
        load_vae_checkpoint(tr.vae, load_path)

    dataloader = create_dataloader(dataset_url, batch_size, num_workers=4, do_shuffle=True)
    test_dataloader = create_dataloader(test_dataset_url, batch_size, num_workers=4, do_shuffle=False, just_resize=True)
    if isinstance(dataloader, SyntheticLoader) and not decoder_also_perform_hr:
        dataloader = SyntheticLoader(batch_size, 256)  # 256^2 "hr" images: the only shape-consistent non-HR recipe
    if isinstance(test_dataloader, SyntheticLoader):
        test_dataloader = SyntheticLoader(batch_size, 512 if decoder_also_perform_hr else 256, seed=7, n_distinct=2)
    t0 = time.time()
    done = False
    for epoch in range(num_epochs):
        for i, batch in enumerate(dataloader):
            time_taken_till_load = time.time() - t0
            t0 = time.time()
            if tr.global_step >= max_steps:
                done = True
                break
            out = tr.step(batch[0])
            step = tr.global_step - 1
            time_taken_till_step = time.time() - t0
            if master_process and step % 5 == 0:
                ld = out["loss_data"]
                items = [("perceptual_loss", float(out["perceptual_loss"])), ("mse_loss", float(ld["recon_loss"])),
                         ("kl_loss", float(ld["kl_loss"])), ("overall_vae_loss", float(out["overall_vae_loss"])),
                         ("ABS mu (0.0): average_of_abs_z", float(ld["average_of_abs_z"])),
                         ("STD mu : std_of_abs_z", float(ld["std_of_abs_z"]))]
                items += [(f"z_quantiles/{q}", float(v)) for q, v in tr.z_quantiles(out["z"]).items()]
                items += [("time_taken_till_step", time_taken_till_step), ("time_taken_till_load", time_taken_till_load)]
                if do_ganloss:
                    items = [("d_loss", float(out["d_loss"])), ("gan_loss", float(out["g_gan_loss"])),
                             ("avg_real_logits", float(out["avg_real_logits"])),
                             ("avg_fake_logits", float(out["avg_fake_logits"])),
                             ("discriminator_accuracy", float(out["disc_acc"])),
                             ("lecam_loss", float(out["lecam_loss"])),
                             ("lecam_anchor_real_logits", float(tr.lecam_anchor_real_logits)),
                             ("lecam_anchor_fake_logits", float(tr.lecam_anchor_fake_logits))] + items
                logger.info(f"Epoch [{epoch}/{num_epochs}] step {step} - " +
                            "\n\t".join(f"{k}: {v:.4f}" for k, v in items))
                if use_wandb:
                    wandb.log({k: v for k, v in items})
            t0 = time.time()
            if evaluate_every_n_steps > 0 and tr.global_step % evaluate_every_n_steps == 1 and master_process:
                ev = tr.evaluate(test_dataloader)  # :811-893: reconstruction grids of (up to) 8 test images
                logger.info(f"Epoch [{epoch}/{num_epochs}] - Logging test images")
                if use_wandb:
                    wandb.log({"reconstructed_test_images": [wandb.Image(ev["reconstructed_test_images"])],
                               "test_images": [wandb.Image(ev["test_images"])]})
                os.makedirs(f"./ckpt/{run_name}", exist_ok=True)  # :903-910: VAE weights only, DDP-prefixed keys
                ck = f"./ckpt/{run_name}/vae_epoch_{epoch}_step_{tr.global_step}.pt"
                torch.save(tr.vae.state_dict(), ck)
                print(f"Saved checkpoint to {ck}")
        if done:
            break
    tr.release_graph()  # a live CUDA graph holds NCCL work: release it before the process group goes away
    cleanup()


if __name__ == "__main__":
    # Example: torchrun --nproc_per_node=8 vae_trainer.py --vae_ch 128 --do_clamp --batch_size 16 --max_steps 100
    train_ddp()
