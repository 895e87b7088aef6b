"""The 3-D PatchGAN discriminator of video training (tae_disc.PatchDiscriminator3D), in plain PyTorch.

The reference has no video discriminator, so this module is its definition (DESIGN.md section 7 row 24): the
NLayerDiscriminator topology built from the TVAE's own conv geometries, convolving over time as well as space. With
m_i = min(2^i, 8):

  conv_in                       F.pad(x, (0,1,0,1,0,1)), Conv3d(3, ch, 3, stride 2) with bias, LeakyReLU(0.2)     /2
  down.{i-1}, i < n_layers      pad as above, Conv3d(ch m_{i-1}, ch m_i, 3, stride 2, no bias), GroupNorm(32, eps
                                1e-6), LeakyReLU(0.2)                                                            /2 each
  mid                           Conv3d(ch m_{n-1}, ch m_n, 3, padding 1, no bias), GroupNorm(32), LeakyReLU(0.2)
  conv_out                      Conv3d(ch m_n, 1, 3, padding 1) with bias           -> [B, 1, T/2^n, H/2^n, W/2^n]

forward(x) returns the logits flattened to [B, L]. The input is the raw clip in the TVAE's range (no ScalingLayer:
there is no pretrained trunk). Init: conv weights N(0, 0.02), conv biases 0, GroupNorm weight 1 and bias 0. The
parameter names are tae_disc.PatchDiscriminator3D's, so state dicts load both ways. TEST INFRASTRUCTURE (see
oracle/__init__.py) and the eager peer of tools/tae_loss_bench.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

LEAKY_SLOPE = 0.2


def channel_plan(ch: int, n_layers: int, in_channels: int = 3):
    """-> [(Cin, Cout, stride)] of the n_layers + 2 convolutions, conv_in first and conv_out last."""
    m = [min(2 ** i, 8) for i in range(n_layers + 1)]
    plan = [(in_channels, ch, 2)]
    plan += [(ch * m[i - 1], ch * m[i], 2) for i in range(1, n_layers)]
    plan += [(ch * m[n_layers - 1], ch * m[n_layers], 1), (ch * m[n_layers], 1, 1)]
    return plan


class _ConvNorm(nn.Module):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv = nn.Conv3d(cin, cout, 3, stride=stride, padding=1 if stride == 1 else 0, bias=False)
        self.norm = nn.GroupNorm(32, cout, eps=1e-6)

    def forward(self, x):
        if self.conv.stride[0] == 2:
            x = F.pad(x, (0, 1, 0, 1, 0, 1))
        return F.leaky_relu(self.norm(self.conv(x)), LEAKY_SLOPE)


class PatchDiscriminator3D(nn.Module):
    def __init__(self, in_channels: int = 3, ch: int = 64, n_layers: int = 3):
        super().__init__()
        plan = channel_plan(ch, n_layers, in_channels)
        self.conv_in = nn.Conv3d(in_channels, ch, 3, stride=2)
        self.down = nn.ModuleList([_ConvNorm(*p) for p in plan[1:n_layers]])
        self.mid = _ConvNorm(*plan[n_layers])
        self.conv_out = nn.Conv3d(plan[-1][0], 1, 3, padding=1)
        init_weights(self)

    def forward(self, x):
        h = F.leaky_relu(self.conv_in(F.pad(x, (0, 1, 0, 1, 0, 1))), LEAKY_SLOPE)
        for blk in self.down:
            h = blk(h)
        return self.conv_out(self.mid(h)).flatten(1)


def init_weights(module: nn.Module):
    """Conv weights N(0, 0.02), conv biases 0, GroupNorm weight 1 and bias 0 (the PatchGAN initialisation)."""
    for m in module.modules():
        if isinstance(m, nn.Conv3d):
            nn.init.normal_(m.weight, 0.0, 0.02)
            if m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.GroupNorm):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)


def forward(sd: dict, x: torch.Tensor, n_layers: int) -> torch.Tensor:
    """Functional form on a state_dict (the tensors may require grad, or be detached to freeze D): -> [B, L]."""
    pad = lambda t: F.pad(t, (0, 1, 0, 1, 0, 1))  # noqa: E731
    h = F.leaky_relu(F.conv3d(pad(x), sd["conv_in.weight"], sd["conv_in.bias"], stride=2), LEAKY_SLOPE)
    blocks = [(f"down.{i}", 2) for i in range(n_layers - 1)] + [("mid", 1)]
    for p, stride in blocks:
        h = F.conv3d(pad(h) if stride == 2 else h, sd[f"{p}.conv.weight"], None, stride=stride,
                     padding=0 if stride == 2 else 1)
        h = F.leaky_relu(F.group_norm(h, 32, sd[f"{p}.norm.weight"], sd[f"{p}.norm.bias"], 1e-6), LEAKY_SLOPE)
    return F.conv3d(h, sd["conv_out.weight"], sd["conv_out.bias"], padding=1).flatten(1)


def flops(ch: int, n_layers: int, B: int, T: int, H: int, W: int, only_first: bool = False) -> int:
    """Multiply-adds x 2 of one forward's convolutions (27 taps per output voxel and channel pair), from the shapes;
    only_first: conv_in's alone."""
    total, t, h, w = 0, T, H, W
    for cin, cout, stride in channel_plan(ch, n_layers)[:1 if only_first else None]:
        t, h, w = t // stride, h // stride, w // stride
        total += 2 * 27 * cin * cout * B * t * h * w
    return total
