"""H100-native drop-in for the reference `tae.py` (TVAE, the video autoencoder): no-grad inference, and training once
opted in with `enable_training`.

Same names, constructor signatures, parameter creation order (so `torch.manual_seed(s); TVAE(...)` yields the
reference's initial weights bit for bit), `state_dict` keys and OIDHW shapes, and return values as the reference; no
einops. Every forward runs hand-written sm_90a kernels (libvqb200.so):

  3x3x3 convs (stride 1, and the (0,1,0,1,0,1)-padded stride-2 Downsample) -> 5-D TMA implicit-GEMM wgmma kernel
                                                                              (vqb_conv3d_gemm)
  Upsample (nearest x2 in T, H, W + 3x3x3 conv)                            -> eight 2x2x2-tap phase convs over the
                                                                              low-resolution input (8/27 of the MACs)
  1x1x1 convs (nin_shortcut, qkv, proj_out)                               -> vqb_conv_gemm on the [N][T*H][W][C] view
  GroupNorm(+swish)                                                        -> the GroupNorm kernels over T*H*W voxels
  AttnBlock core (8 heads of C/8 channels)                                 -> flash-style kernel, heads of 8 to 112
                                                                              channels in steps of 8
  DiagonalGaussian                                                         -> torch.randn_like(mean) + one fused kernel

Internally activations are bf16 NTHWC (`Act3`); modules accept an `Act3` or an NCTHW tensor and return NCTHW in the
dtype of their parameters (fp32 or bf16).

Training is opted into explicitly: `tae.enable_training(vae)` (returns vae). Then a grad-enabled forward records the
autograd functions of ops.py (Conv3dFn, UpConv3dFn, GroupNormSiLUFn, AttentionHdFn, GaussReparamFn), whose backward runs
the 3-D data- and weight-gradient kernels; parameters may be frozen and the input may require grad (the gradient of the
video). Without the opt-in, a forward that autograd would have to differentiate (grad enabled and parameters that
require grad) raises before anything is launched: a grad-enabled forward of a full clip would otherwise keep many GB of
activations alive. `tae.enable_training(vae, recompute=True)` bounds that memory: each ResnetBlock then keeps only its
input for the backward (ops.ResnetBlock3dRecomputeFn) and rebuilds hn, h and h2 there bit for bit, so the gradients
are those of the plain path. Modules with bf16 parameters stay inference-only. Deviations from the reference (DESIGN.md
section 7): training is opt-in; T, H and W divisible by 2^(len(ch_mult)-1) at the encoder; heads of 8 to 112
channels in steps of 8 (C a multiple of 64 up to 896).

Reference citations: tae.py:9-10 swish, :13-54 AttnBlock, :57-90 ResnetBlock, :93-104 Downsample, :107-117 Upsample,
:120-184 Encoder, :187-250 Decoder, :253-266 DiagonalGaussian, :269-297 TVAE.
"""
from __future__ import annotations

import contextlib
import math
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import torch
from torch import Tensor, nn

import ops
import plans


class Act3:
    """Internal activation: bf16 NTHWC tensor `t` [N, T, H, W, Cp] carrying its true channel count `C`."""

    __slots__ = ("t", "C")

    def __init__(self, t: Tensor, C: int):
        self.t = t
        self.C = C

    @property
    def shape(self):  # reference-style (N, C, T, H, W)
        n, t, h, w, _ = self.t.shape
        return (n, self.C, t, h, w)


def _param_dtype(module: nn.Module):
    """dtype of the module's parameters (fp32 or bf16); other dtypes raise here, before anything is launched."""
    p = next(module.parameters(), None)
    if p is None:
        return torch.float32
    ops.check_master_dtype(p, f"{type(module).__name__} parameter")
    return p.dtype


def enable_training(module: nn.Module, enabled: bool = True, recompute: bool = False) -> nn.Module:
    """Opts `module` and every submodule into training (enabled=False opts out again and clears `recompute`); returns
    `module`.

    Once opted in, a grad-enabled forward records for autograd and `loss.backward()` runs the native 3-D gradient
    kernels; no-grad forwards are unchanged. Parameters must be float32 (bf16 modules are inference-only).
    recompute=True makes every ResnetBlock under `module` keep only its input (plus two [N, 32, 2] GroupNorm records)
    for the backward and rebuild its three inner activations there, bit for bit: less activation memory for one extra
    conv1 and two GroupNorm apply passes per block in the backward. Gradients equal the non-recomputing path's."""
    for m in module.modules():
        m._vqb_training = bool(enabled)
        if isinstance(m, ResnetBlock):
            m._vqb_recompute = bool(enabled and recompute)
    return module


def _opted_in(module: nn.Module) -> bool:
    return getattr(module, "_vqb_training", False)


def _grad_path(module: nn.Module) -> bool:
    """True when this forward records for autograd: grad enabled and the module opted in."""
    return torch.is_grad_enabled() and _opted_in(module)


def _mode(module: nn.Module):
    """The forward's autograd context: recording on the training path, torch.no_grad() otherwise."""
    return contextlib.nullcontext() if _grad_path(module) else torch.no_grad()


def _check_trainable(module: nn.Module):
    for p in module.parameters():
        if p.dtype != torch.float32:
            raise RuntimeError(
                f"vqgan-training_b200: tae.{type(module).__name__} has {p.dtype} parameters; training needs float32 "
                "master weights (bf16 modules are inference-only). Run it under torch.no_grad() / "
                "torch.inference_mode(), or train the float32 module (`.float()`).")


def _inference_only(module: nn.Module):
    if _grad_path(module):
        _check_trainable(module)
        return
    if torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters()):
        raise RuntimeError(
            f"vqgan-training_b200: tae.{type(module).__name__} runs inference only unless opted into training: run it "
            "under torch.no_grad() / torch.inference_mode(), freeze its parameters (requires_grad_(False)), or call "
            "tae.enable_training(module) to train it.")


def _enter(x, module: nn.Module):
    """NCTHW tensor -> Act3 (or pass an Act3 through). Returns (act, was_external)."""
    if isinstance(x, Act3):
        return x, False
    _inference_only(module)
    _param_dtype(module)
    if x.dim() != 5:
        raise ValueError(f"tae.{type(module).__name__}: expected an NCTHW tensor, got shape {tuple(x.shape)}")
    ops.require_cuda(x)
    N, C, T, H, W = x.shape
    if _grad_path(module):  # the input may require grad (the gradient of the video)
        y = ops.to_nhwc(x.reshape(N, C, T * H, W))
    else:
        y = ops.to_nhwc(x.detach().reshape(N, C, T * H, W))
    return Act3(y.view(N, T, H, W, y.shape[-1]), C), True


def _exit(a: Act3, external: bool, module: nn.Module):
    if not external:
        return a
    N, T, H, W, Cp = a.t.shape
    y = ops.to_nchw(a.t.view(N, T * H, W, Cp), a.C, _param_dtype(module))
    return y.view(N, a.C, T, H, W)


def swish(x: Tensor) -> Tensor:
    """tae.py:9-10. On plain tensors this is the reference expression; inside the network it is fused into GroupNorm."""
    if isinstance(x, Act3):
        raise RuntimeError("swish on internal activations is fused into the GroupNorm kernels")
    return x * torch.sigmoid(x)


class Conv3d(nn.Conv3d):
    """nn.Conv3d parameters and initialisation with the native forward (3x3x3 stride 1 or 2, 1x1x1)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._packed = ops.PackedCache()

    def _kind(self):
        k, s, p = self.kernel_size, self.stride, self.padding
        if k == (3, 3, 3) and s == (1, 1, 1) and p == (1, 1, 1):
            return "s1"
        if k == (1, 1, 1) and s == (1, 1, 1) and p == (0, 0, 0):
            return "p1"
        if k == (3, 3, 3) and s == (2, 2, 2) and p == (0, 0, 0):
            return "s2"  # used after Downsample's (0,1,0,1,0,1) zero pad, folded into the TMA zero fill
        raise NotImplementedError(f"Conv3d k={k} s={s} p={p} is not on the native path")

    def forward_act(self, a: Act3, residual: Act3 = None, ncthw_out=False):
        # grad is enabled here only on the training path (the inference path runs under torch.no_grad())
        conv = ops.conv3d_train if torch.is_grad_enabled() else ops.conv3d
        out = conv(a.t, self.weight, self.bias, self._packed, self._kind(),
                   residual.t if residual is not None else None, ncthw_out)
        return out if ncthw_out else Act3(out, self.out_channels)

    def forward(self, x):
        if isinstance(x, Act3):
            return self.forward_act(x)
        if self._kind() == "s2":
            raise RuntimeError("stride-2 Conv3d is only reachable through Downsample")
        a, ext = _enter(x, self)
        with _mode(self):
            return _exit(self.forward_act(a), ext, self)


def _norm(gn: nn.GroupNorm, a: Act3, silu: bool) -> Act3:
    return Act3(ops.group_norm_silu3d(a.t, gn.weight, gn.bias, gn.num_groups, gn.eps, silu), a.C)


def _norm_skip(gn: nn.GroupNorm, a: Act3, silu: bool):
    """Training path: GroupNorm(+swish) that also returns its input as the skip connection, so the skip's gradient is
    summed into dx inside the GroupNorm backward kernel (GroupNormSiLUFn with_skip)."""
    N, T, H, W, C = a.t.shape
    y, skip = ops.group_norm_silu(a.t.reshape(N, T * H, W, C), gn.weight, gn.bias, gn.num_groups, gn.eps, silu,
                                  with_skip=True)
    return Act3(y.view(N, T, H, W, C), a.C), Act3(skip.view(N, T, H, W, C), a.C)


class AttnBlock(nn.Module):
    def __init__(self, in_channels: int):
        super().__init__()
        self.in_channels = in_channels
        self.num_heads = 8
        self.head_dim = in_channels // self.num_heads
        self.norm = nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)
        self.qkv = Conv3d(in_channels, in_channels * 3, kernel_size=1, bias=False)
        self.proj_out = Conv3d(in_channels, in_channels, kernel_size=1, bias=False)
        nn.init.normal_(self.proj_out.weight, std=0.2 / math.sqrt(in_channels))

    def _check_heads(self):
        if self.head_dim not in ops.ATTN_HEAD_DIMS or self.head_dim * self.num_heads != self.in_channels:
            raise NotImplementedError(
                f"tae.AttnBlock({self.in_channels}): heads of {self.in_channels / self.num_heads:g} channels are not "
                "supported (heads of 8 to 112 channels in steps of 8 only: in_channels a multiple of 64 up to 896)")

    def attention(self, h_) -> Act3:
        self._check_heads()
        a, ext = _enter(h_, self)
        with _mode(self):
            qkv = self.qkv.forward_act(_norm(self.norm, a, silu=False))
            attn = ops.attention_hd_train if torch.is_grad_enabled() else ops.attention_hd
            o = Act3(attn(qkv.t, self.num_heads, self.head_dim), self.in_channels)
            return _exit(o, ext, self)

    def forward(self, x):
        self._check_heads()
        a, ext = _enter(x, self)
        with _mode(self):
            if torch.is_grad_enabled():  # training path
                hn, skip = _norm_skip(self.norm, a, silu=False)
                qkv = self.qkv.forward_act(hn)
                h = Act3(ops.attention_hd_train(qkv.t, self.num_heads, self.head_dim), self.in_channels)
                return _exit(self.proj_out.forward_act(h, residual=skip), ext, self)
            h = self.attention(a)
            out = self.proj_out.forward_act(h, residual=a)  # x + proj_out(attention(x)) fused in the conv epilogue
            return _exit(out, ext, self)


class ResnetBlock(nn.Module):
    def __init__(self, in_channels: int, out_channels: int = None):
        super().__init__()
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.norm1 = nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)
        self.conv1 = Conv3d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = nn.GroupNorm(num_groups=32, num_channels=out_channels, eps=1e-6, affine=True)
        self.conv2 = Conv3d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            self.nin_shortcut = Conv3d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

    def _recompute(self, a: Act3) -> Act3:
        """Training path of enable_training(..., recompute=True): the block as one autograd node that saves only x."""
        nin = self.nin_shortcut if self.in_channels != self.out_channels else None
        spec = (self.norm1.num_groups, self.norm1.eps, self.norm2.num_groups, self.norm2.eps, self.conv1._packed,
                self.conv2._packed, nin._packed if nin is not None else None)
        out = ops.resnet_block3d_recompute(
            a.t, spec, self.norm1.weight, self.norm1.bias, self.conv1.weight, self.conv1.bias, self.norm2.weight,
            self.norm2.bias, self.conv2.weight, self.conv2.bias, nin.weight if nin is not None else None,
            nin.bias if nin is not None else None)
        return Act3(out, self.out_channels)

    def forward(self, x):
        a, ext = _enter(x, self)
        with _mode(self):
            if torch.is_grad_enabled() and getattr(self, "_vqb_recompute", False):
                return _exit(self._recompute(a), ext, self)
            if torch.is_grad_enabled():  # training path
                hn, skip = _norm_skip(self.norm1, a, silu=True)
                h = self.conv1.forward_act(hn)
                h = _norm(self.norm2, h, silu=True)
                skip = self.nin_shortcut.forward_act(skip) if self.in_channels != self.out_channels else skip
                return _exit(self.conv2.forward_act(h, residual=skip), ext, self)
            h = self.conv1.forward_act(_norm(self.norm1, a, silu=True))
            h = _norm(self.norm2, h, silu=True)
            skip = self.nin_shortcut.forward_act(a) if self.in_channels != self.out_channels else a
            out = self.conv2.forward_act(h, residual=skip)  # x + h fused in the conv epilogue
            return _exit(out, ext, self)


def _check_even(shape, what):
    N, C, T, H, W = shape
    if T % 2 or H % 2 or W % 2:
        raise ValueError(f"tae.{what}: T, H and W must be even at every Downsample; got (T, H, W) = ({T}, {H}, {W}) "
                         f"for input shape {tuple(shape)}")


class Downsample(nn.Module):
    def __init__(self, in_channels: int):
        super().__init__()
        self.conv = Conv3d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def forward(self, x: Tensor):
        # F.pad(x, (0,1,0,1,0,1)) + stride-2 conv (tae.py:100-104): the pad planes are the TMA unit's zero fill
        _check_even(tuple(x.shape), "Downsample")
        a, ext = _enter(x, self)
        with _mode(self):
            return _exit(self.conv.forward_act(a), ext, self)


class Upsample(nn.Module):
    def __init__(self, in_channels: int):
        super().__init__()
        self.conv = Conv3d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x: Tensor):
        # nearest x2 + 3x3x3 conv as eight 2x2x2-tap phase convs over the low-resolution tensor
        a, ext = _enter(x, self)
        with _mode(self):
            up = ops.upsample_conv3d_train if torch.is_grad_enabled() else ops.upsample_conv3d
            y = up(a.t, self.conv.weight, self.conv.bias, self.conv._packed)
            return _exit(Act3(y, self.conv.out_channels), ext, self)


class Encoder(nn.Module):
    def __init__(
        self,
        resolution: int,
        in_channels: int,
        ch: int,
        ch_mult: list[int],
        num_res_blocks: int,
        z_channels: int,
    ):
        super().__init__()
        self.ch = ch
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.conv_in = Conv3d(in_channels, self.ch, kernel_size=3, stride=1, padding=1)
        curr_res = resolution
        in_ch_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        block_in = self.ch
        for i_level in range(self.num_resolutions):
            block = nn.ModuleList()
            attn = nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out))
                block_in = block_out
            down = nn.Module()
            down.block = block
            down.attn = attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in)
        self.norm_out = nn.GroupNorm(num_groups=32, num_channels=block_in, eps=1e-6, affine=True)
        self.conv_out = Conv3d(block_in, 2 * z_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x: Tensor) -> Tensor:
        f = 2 ** (self.num_resolutions - 1)
        if x.dim() != 5 or any(s % f for s in x.shape[2:]):
            raise ValueError(f"tae.Encoder: T, H and W must be divisible by {f} (even at each of the "
                             f"{self.num_resolutions - 1} Downsample levels); got input shape {tuple(x.shape)}")
        self.mid.attn_1._check_heads()
        a, _ = _enter(x, self)
        with _mode(self):
            a = self.conv_in.forward_act(a)
            for i_level in range(self.num_resolutions):
                for i_block in range(self.num_res_blocks):
                    a = self.down[i_level].block[i_block](a)
                    if len(self.down[i_level].attn) > 0:
                        a = self.down[i_level].attn[i_block](a)
                if i_level != self.num_resolutions - 1:
                    a = self.down[i_level].downsample(a)
            a = self.mid.block_1(a)
            a = self.mid.attn_1(a)
            a = self.mid.block_2(a)
            a = _norm(self.norm_out, a, silu=True)
            return self.conv_out.forward_act(a, ncthw_out=True)  # [N, 2*z_channels, T/f, H/f, W/f]


class Decoder(nn.Module):
    def __init__(
        self,
        ch: int,
        out_ch: int,
        ch_mult: list[int],
        num_res_blocks: int,
        in_channels: int,
        resolution: int,
        z_channels: int,
    ):
        super().__init__()
        self.ch = ch
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.ffactor = 2 ** (self.num_resolutions - 1)
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // (2 ** (self.num_resolutions - 1))
        self.z_shape = (1, z_channels, curr_res, curr_res, curr_res)
        self.conv_in = Conv3d(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block = nn.ModuleList()
            attn = nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks + 1):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out))
                block_in = block_out
            up = nn.Module()
            up.block = block
            up.attn = attn
            if i_level != 0:
                up.upsample = Upsample(block_in)
                curr_res = curr_res * 2
            self.up.insert(0, up)
        self.norm_out = nn.GroupNorm(num_groups=32, num_channels=block_in, eps=1e-6, affine=True)
        self.conv_out = Conv3d(block_in, out_ch, kernel_size=3, stride=1, padding=1)

    def forward(self, z: Tensor) -> Tensor:
        self.mid.attn_1._check_heads()
        a, _ = _enter(z, self)
        with _mode(self):
            a = self.conv_in.forward_act(a)
            a = self.mid.block_1(a)
            a = self.mid.attn_1(a)
            a = self.mid.block_2(a)
            for i_level in reversed(range(self.num_resolutions)):
                for i_block in range(self.num_res_blocks + 1):
                    a = self.up[i_level].block[i_block](a)
                    if len(self.up[i_level].attn) > 0:
                        a = self.up[i_level].attn[i_block](a)
                if i_level != 0:
                    a = self.up[i_level].upsample(a)
            a = _norm(self.norm_out, a, silu=True)
            return self.conv_out.forward_act(a, ncthw_out=True)  # [N, out_ch, T, H, W]


class DiagonalGaussian(nn.Module):
    def __init__(self, sample: bool = True, chunk_dim: int = 1):
        super().__init__()
        self.sample = sample
        self.chunk_dim = chunk_dim

    def forward(self, z: Tensor) -> Tensor:
        mean, logvar = torch.chunk(z, 2, dim=self.chunk_dim)
        if not self.sample:
            return mean
        if self.chunk_dim != 1:
            raise NotImplementedError("tae.DiagonalGaussian: the native sampler takes chunk_dim=1 (channels)")
        if torch.is_grad_enabled() and z.requires_grad:
            if not _opted_in(self):
                raise RuntimeError("vqgan-training_b200: tae.DiagonalGaussian runs inference only unless opted into "
                                   "training: run it under torch.no_grad() / torch.inference_mode(), or call "
                                   "tae.enable_training(module)")
            if z.dtype != torch.float32:
                raise RuntimeError(f"vqgan-training_b200: tae.DiagonalGaussian: training needs a float32 latent, got "
                                   f"{z.dtype} (bf16 modules are inference-only)")
            eps = torch.randn_like(mean)  # the reference's own draw (tae.py:264)
            return ops.gauss_reparam_train(z, eps)
        # the reference's own draw (tae.py:264): a seeded run consumes the same RNG stream and gets the same eps
        eps = torch.randn_like(mean)
        return ops.gauss_reparam(z, eps)


class TVAE(nn.Module):
    def __init__(
        self, resolution, in_channels, ch, out_ch, ch_mult, num_res_blocks, z_channels
    ):
        super().__init__()
        self.encoder = Encoder(
            resolution=resolution,
            in_channels=in_channels,
            ch=ch,
            ch_mult=ch_mult,
            num_res_blocks=num_res_blocks,
            z_channels=z_channels,
        )
        self.decoder = Decoder(
            resolution=resolution,
            in_channels=in_channels,
            ch=ch,
            out_ch=out_ch,
            ch_mult=ch_mult,
            num_res_blocks=num_res_blocks,
            z_channels=z_channels,
        )
        self.reg = DiagonalGaussian()

    def forward(self, x: Tensor) -> Tensor:
        if _grad_path(self):
            _check_trainable(self)  # a bf16 part is refused before the encoder launches anything
        z = self.encoder(x)
        z_s = self.reg(z)
        decz = self.decoder(z_s)
        return decz, z
