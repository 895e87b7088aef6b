"""Functional restatement of the reference video autoencoder (tae.py, TVAE) from its semantics: F.conv3d,
F.group_norm, an explicit softmax attention and F.interpolate over a reference-format state_dict. Runs in the dtype of
the state_dict / input it is given (fp32 truth, or bf16 for the model-card-style peer).

    z    = encoder_forward(sd, x, cfg)          # [N, 2*z_channels, T/f, H/f, W/f]
    z_s  = reg(z, eps)                          # mean + exp(0.5 * logvar.clamp(min=-3)) * eps
    decz = decoder_forward(sd, z_s, cfg)        # [N, out_ch, T, H, W]
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple

import torch
import torch.nn.functional as F


@dataclass
class TAEConfig:
    ch: int = 64
    ch_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 16
    in_channels: int = 3
    out_ch: int = 3
    resolution: int = 256

    def kwargs(self):
        """Constructor arguments of TVAE."""
        return dict(resolution=self.resolution, in_channels=self.in_channels, ch=self.ch, out_ch=self.out_ch,
                    ch_mult=list(self.ch_mult), num_res_blocks=self.num_res_blocks, z_channels=self.z_channels)


def _conv(sd, p, x, stride=1, padding=1):
    return F.conv3d(x, sd[p + ".weight"], sd.get(p + ".bias"), stride=stride, padding=padding)


def _gn(sd, p, x):
    return F.group_norm(x, 32, sd[p + ".weight"], sd[p + ".bias"], eps=1e-6)


def _swish(x):
    return x * torch.sigmoid(x)


def resnet_block(sd, p, x):
    h = _conv(sd, p + ".conv1", _swish(_gn(sd, p + ".norm1", x)))
    h = _conv(sd, p + ".conv2", _swish(_gn(sd, p + ".norm2", h)))
    if p + ".nin_shortcut.weight" in sd:
        x = _conv(sd, p + ".nin_shortcut", x, padding=0)
    return x + h


def attn_block(sd, p, x, heads=8):
    N, C, T, H, W = x.shape
    d = C // heads
    qkv = _conv(sd, p + ".qkv", _gn(sd, p + ".norm", x), padding=0)
    q, k, v = (t.reshape(N, heads, d, T * H * W).transpose(-1, -2) for t in qkv.chunk(3, dim=1))
    a = torch.softmax((q @ k.transpose(-1, -2)) * d ** -0.5, dim=-1)
    o = (a @ v).transpose(-1, -2).reshape(N, C, T, H, W)
    return x + _conv(sd, p + ".proj_out", o, padding=0)


def encoder_forward(sd, x, cfg: TAEConfig):
    p = "encoder."
    h = _conv(sd, p + "conv_in", x)
    n = len(cfg.ch_mult)
    for i in range(n):
        for b in range(cfg.num_res_blocks):
            h = resnet_block(sd, f"{p}down.{i}.block.{b}", h)
        if i != n - 1:
            h = _conv(sd, f"{p}down.{i}.downsample.conv", F.pad(h, (0, 1, 0, 1, 0, 1)), stride=2, padding=0)
    h = resnet_block(sd, p + "mid.block_1", h)
    h = attn_block(sd, p + "mid.attn_1", h)
    h = resnet_block(sd, p + "mid.block_2", h)
    return _conv(sd, p + "conv_out", _swish(_gn(sd, p + "norm_out", h)))


def decoder_forward(sd, z, cfg: TAEConfig):
    p = "decoder."
    h = _conv(sd, p + "conv_in", z)
    h = resnet_block(sd, p + "mid.block_1", h)
    h = attn_block(sd, p + "mid.attn_1", h)
    h = resnet_block(sd, p + "mid.block_2", h)
    for i in reversed(range(len(cfg.ch_mult))):
        for b in range(cfg.num_res_blocks + 1):
            h = resnet_block(sd, f"{p}up.{i}.block.{b}", h)
        if i != 0:
            h = _conv(sd, f"{p}up.{i}.upsample.conv", F.interpolate(h, scale_factor=2.0, mode="nearest"))
    return _conv(sd, p + "conv_out", _swish(_gn(sd, p + "norm_out", h)))


def reg(z, eps):
    """DiagonalGaussian with sample=True, the noise given: mean + exp(0.5 * logvar.clamp(min=-3)) * eps."""
    mean, logvar = z.chunk(2, dim=1)
    return mean + torch.exp(0.5 * logvar.clamp(min=-3)) * eps


def forward(sd, x, eps, cfg: TAEConfig):
    """TVAE.forward with the noise given -> (decz, z)."""
    z = encoder_forward(sd, x, cfg)
    return decoder_forward(sd, reg(z, eps), cfg), z


def flops(cfg: TAEConfig, N, T, H, W, infer="reconstruct"):
    """Algorithmic multiply-add FLOPs (2 per MAC) of the forward as the plans execute it: 3x3x3 convs, the folded
    up-sampling (8 phases of 2x2x2 taps over the low-resolution grid), 1x1x1 convs and the attention matmuls.
    GroupNorm, softmax and elementwise work are not counted."""
    tot = {"encoder": 0, "decoder": 0}

    def conv(part, cin, cout, taps, vox):
        tot[part] += 2 * cin * cout * taps * vox * N

    n = len(cfg.ch_mult)
    ch = cfg.ch
    vox = T * H * W
    # encoder
    conv("encoder", cfg.in_channels, ch, 27, vox)
    cin = ch
    for i in range(n):
        cout = ch * cfg.ch_mult[i]
        for _ in range(cfg.num_res_blocks):
            conv("encoder", cin, cout, 27, vox)
            conv("encoder", cout, cout, 27, vox)
            if cin != cout:
                conv("encoder", cin, cout, 1, vox)
            cin = cout
        if i != n - 1:
            vox //= 8
            conv("encoder", cin, cin, 27, vox)

    def mid(part, c, v):
        for _ in range(2):
            conv(part, c, c, 27, v)
            conv(part, c, c, 27, v)
        conv(part, c, 3 * c, 1, v)
        conv(part, c, c, 1, v)
        tot[part] += 2 * 2 * v * v * c * N  # q k^T and p v over all heads

    mid("encoder", cin, vox)
    conv("encoder", cin, 2 * cfg.z_channels, 27, vox)
    # decoder
    cin = ch * cfg.ch_mult[-1]
    conv("decoder", cfg.z_channels, cin, 27, vox)
    mid("decoder", cin, vox)
    for i in reversed(range(n)):
        cout = ch * cfg.ch_mult[i]
        for _ in range(cfg.num_res_blocks + 1):
            conv("decoder", cin, cout, 27, vox)
            conv("decoder", cout, cout, 27, vox)
            if cin != cout:
                conv("decoder", cin, cout, 1, vox)
            cin = cout
        if i != 0:
            conv("decoder", cin, cin, 8 * 8, vox)  # 8 phases x 8 folded taps over the low-resolution grid
            vox *= 8
    conv("decoder", cin, cfg.out_ch, 27, vox)
    if infer == "encode":
        return tot["encoder"]
    if infer == "decode":
        return tot["decoder"]
    return tot["encoder"] + tot["decoder"]
