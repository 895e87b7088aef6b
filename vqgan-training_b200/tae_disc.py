"""3-D PatchGAN discriminator for video autoencoder training, on the native 3-D kernels of tae.py.

The per-frame PatchDiscriminator (utils.py) scores frames one at a time, so it never sees two frames together. This
discriminator convolves over time as well as space (DESIGN.md section 7 row 24; oracle/clip_disc_oracle.py is its
plain-PyTorch definition, with the same parameter names, so state dicts load both ways). With m_i = min(2^i, 8):

  conv_in                       (0,1,0,1,0,1)-padded 3x3x3 stride-2 conv with bias, LeakyReLU(0.2)         /2
  down.{i-1}, i < n_layers      padded stride-2 conv without bias, GroupNorm(32, eps 1e-6) + LeakyReLU(0.2) /2 each
  mid                           3x3x3 padding-1 conv without bias, GroupNorm(32) + LeakyReLU(0.2)
  conv_out                      3x3x3 padding-1 conv to one channel with bias   -> logits [B, (T/2^n)(H/2^n)(W/2^n)]

The convolutions are the TVAE's (tae.Conv3d: Downsample's stride-2 geometry and the stride-1 one), GroupNorm and its
LeakyReLU are one fused pass (activation code 2 of the GroupNorm kernels), and conv_in's LeakyReLU is a standalone
vectorised pass (ops.leaky_relu). The input is the raw clip in the TVAE's range: there is no ScalingLayer.

A no-grad forward needs no opt-in. Training is opted into with tae.enable_training(disc) (VideoTrainer does it); then
the parameters may be frozen and the clip may require grad (the generator pass). bf16 modules are inference-only.
"""
from __future__ import annotations

import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import torch
from torch import Tensor, nn

import ops
import tae
from tae import Act3


class _ConvNorm(nn.Module):
    """A bias-free 3x3x3 conv (stride 2 after the (0,1,0,1,0,1) pad, or stride 1 with padding 1), then GroupNorm(32)
    fused with LeakyReLU(0.2)."""

    def __init__(self, cin: int, cout: int, stride: int):
        super().__init__()
        self.conv = tae.Conv3d(cin, cout, kernel_size=3, stride=stride, padding=1 if stride == 1 else 0, bias=False)
        self.norm = nn.GroupNorm(num_groups=32, num_channels=cout, eps=1e-6, affine=True)

    def forward_act(self, a: Act3) -> Act3:
        a = self.conv.forward_act(a)
        return Act3(ops.group_norm_silu3d(a.t, self.norm.weight, self.norm.bias, self.norm.num_groups, self.norm.eps,
                                          ops.ACT_LEAKY), a.C)


class PatchDiscriminator3D(nn.Module):
    """PatchDiscriminator3D(in_channels=3, ch=64, n_layers=3): forward(x [B, 3, T, H, W]) -> logits [B, L], the shape
    vae_trainer.gan_disc_loss and LeCam take. T, H and W must be divisible by 2^n_layers; ch a multiple of 32 up to
    256 (GroupNorm(32) over at most 8 ch channels, which the GroupNorm kernels take up to 2048)."""

    def __init__(self, in_channels: int = 3, ch: int = 64, n_layers: int = 3):
        super().__init__()
        if n_layers < 1:
            raise ValueError(f"PatchDiscriminator3D: n_layers must be >= 1, got {n_layers}")
        if ch <= 0 or ch % 32 or ch > 256:
            raise ValueError(f"PatchDiscriminator3D: ch must be a multiple of 32 up to 256 (GroupNorm(32) over up to "
                             f"8 ch channels), got {ch}")
        self.in_channels, self.ch, self.n_layers = in_channels, ch, n_layers
        m = [min(2 ** i, 8) for i in range(n_layers + 1)]
        self.conv_in = tae.Conv3d(in_channels, ch, kernel_size=3, stride=2, padding=0)
        self.down = nn.ModuleList([_ConvNorm(ch * m[i - 1], ch * m[i], 2) for i in range(1, n_layers)])
        self.mid = _ConvNorm(ch * m[n_layers - 1], ch * m[n_layers], 1)
        self.conv_out = tae.Conv3d(ch * m[n_layers], 1, kernel_size=3, stride=1, padding=1)
        for mod in self.modules():  # the PatchGAN initialisation (oracle/clip_disc_oracle.py)
            if isinstance(mod, nn.Conv3d):
                nn.init.normal_(mod.weight, 0.0, 0.02)
                if mod.bias is not None:
                    nn.init.zeros_(mod.bias)

    def check_input(self, x: Tensor):
        """The host refusals of forward, raised before anything is launched."""
        if x.dim() != 5 or x.shape[1] != self.in_channels:
            raise ValueError(f"PatchDiscriminator3D: expected a [B, {self.in_channels}, T, H, W] clip, got shape "
                             f"{tuple(x.shape)}")
        f = 2 ** self.n_layers
        if any(s % f for s in x.shape[2:]):
            raise ValueError(f"PatchDiscriminator3D: T, H and W must be divisible by {f} (2^n_layers, n_layers = "
                             f"{self.n_layers}); got clip shape {tuple(x.shape)}")

    def forward(self, x: Tensor) -> Tensor:
        self.check_input(x)
        a, _ = tae._enter(x, self)
        with tae._mode(self):
            a = self.conv_in.forward_act(a)  # kind "s2": the pad planes are the TMA unit's zero fill
            a = Act3(ops.leaky_relu(a.t), a.C)
            for blk in self.down:
                a = blk.forward_act(a)
            a = self.mid.forward_act(a)
            out = self.conv_out.forward_act(a, ncthw_out=True)  # [B, 1, T/2^n, H/2^n, W/2^n], the parameters' dtype
        return out.flatten(1)
