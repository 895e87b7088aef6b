"""H100-native drop-in for the reference `ae.py` (cloneofsimo/vqgan-training): same classes, constructor signatures,
attribute names, parameter creation order (so `torch.manual_seed(s); VAE(...)` yields the reference's init) and
state_dict keys / fp32 OIHW shapes — but every forward/backward runs hand-written sm_90a kernels (libvqb200.so):

  conv 3x3/1x1 s1, Downsample (pad(0,1,0,1)+s2), dgrad, wgrad  -> wgmma implicit-GEMM kernels (csrc/conv_gemm.cu,
                                                                  csrc/wgrad_gemm.cu), TMA-staged, register accumulators
  FP32GroupNorm + swish                                          -> fused stats/apply kernels (csrc/elementwise.cu)
  Upsample (nearest x2) + conv3x3                                -> four 2x2-tap phase convs over the low-res input
  AttnBlock                                                      -> GN kernel + 1x1 conv kernels + flash-style core

Internally activations are bf16 NHWC (`Act`); modules accept either an `Act` (internal) or a plain NCHW tensor
(reference calling convention: converted at the boundary, result returned as NCHW in the dtype of the module's
parameters). Modules converted with `.bfloat16()` run the same kernels from bf16 master weights and return bf16, like
the reference's model-card inference recipe; they are inference-only (a backward through them raises).
`enable_recompute(vae)` bounds training memory: each ResnetBlock then keeps only its input for the backward
(ops.ResnetBlockRecomputeFn) and rebuilds hn, h and h2 there bit for bit.

Reference citations: ae.py:13-14 swish, :41-53 FP32GroupNorm, :56-93 AttnBlock, :96-140 ResnetBlock, :143-154 Downsample,
:157-167 Upsample, :170-257 Encoder, :260-333 Decoder, :336-348 DiagonalGaussian, :351-392 VAE.

Deviations from the reference, all documented in DESIGN.md: (1) `use_attn=True` is constructible (the reference's
bias-zeroing loop crashes on the bias-free attention convs, ae.py:233-235); (2) compute is bf16 with fp32 accumulation in
both encoder and decoder (the reference trains the encoder in TF32 and the decoder under bf16 autocast).
"""
from __future__ import annotations

import math
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import torch
import torch.nn.functional as F
from torch import Tensor, nn

import ops
import plans
from utils import wavelet_transform_multi_channel


class Act:
    """Internal activation: bf16 NHWC tensor `t` [N,H,W,Cp] carrying its true channel count `C`."""

    __slots__ = ("t", "C", "stats", "framed")

    def __init__(self, t: Tensor, C: int, stats=None, framed=False):
        self.t = t
        self.C = C
        self.stats = stats  # per-(n, channel) sum / sum of squares [N, C, 2] when the producing conv computed them
        self.framed = framed  # t is a zero-framed [N, H+2, W+2, 8] image (input of a "fat pixel" first-layer conv)

    @property
    def shape(self):  # reference-style (N, C, H, W)
        n, h, w, _ = self.t.shape
        return (n, self.C, h, w)


def _param_dtype(module: nn.Module):
    """dtype of the module's parameters (fp32, or bf16 for an inference-only module); other dtypes raise here, before
    anything is launched."""
    p = next(module.parameters(), None)
    if p is None:
        return torch.float32
    ops.check_master_dtype(p, f"{type(module).__name__} parameter")
    return p.dtype


def _enter(x, module: nn.Module):
    """NCHW tensor -> Act (or pass an Act through). Returns (act, was_external)."""
    if isinstance(x, Act):
        return x, False
    _param_dtype(module)
    return Act(ops.to_nhwc(x), x.shape[1]), True


def _exit(a: Act, external: bool, module: nn.Module):
    return ops.to_nchw(a.t, a.C, _param_dtype(module)) if external else a


def _stats_fusion() -> bool:
    """Accumulate GroupNorm statistics in the producing conv's epilogue? Its fp32 atomics make the sums' order, and so
    the last bits of every later activation, vary between launches. That is what training pays for one read pass less
    per GroupNorm; without autograd (inference) the statistics come from the GroupNorm's own fixed-order pass instead,
    so the forward is deterministic and a CUDA-graph replay equals the eager run bit for bit."""
    return torch.is_grad_enabled()


def swish(x):
    """ae.py:13-14. On plain tensors this is the reference expression; inside the network it is fused into GroupNorm."""
    if isinstance(x, Act):
        raise RuntimeError("swish on internal activations is fused into FP32GroupNorm.forward(..., silu=True)")
    return x * torch.sigmoid(x)


class StandardizedC2d(nn.Conv2d):
    """nn.Conv2d parameters/initialisation (ae.py:38: StandardizedC2d = nn.Conv2d) with a wgmma forward/backward."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._packed = ops.PackedCache()

    def _kind(self):
        k, s, p = self.kernel_size[0], self.stride[0], self.padding[0]
        if s == 1 and p == (k - 1) // 2:
            return "s1"
        if s == 2 and k == 3 and p == 0:
            return "s2"  # used after the (0,1,0,1) zero pad of Downsample, folded into the kernel's TMA zero fill
        if s == k and p == 0:
            return "patch"
        raise NotImplementedError(f"conv k={k} s={s} p={p} is not on the hot path")

    def forward_act(self, a: Act, residual: Act = None, relu=False, input_is_relu=False, nchw_out=False,
                    want_stats=False):
        """want_stats: also accumulate the GroupNorm statistics of the output in the conv epilogue (Act.stats)."""
        want_stats = want_stats and not nchw_out
        kind = "fat3" if a.framed else self._kind()
        out = ops.conv(a.t, self.weight, self.bias, self._packed, kind,
                       residual.t if residual is not None else None, relu, input_is_relu, nchw_out, want_stats)
        if nchw_out:
            return out
        if want_stats:
            return Act(out[0], self.out_channels, out[1])
        return Act(out, self.out_channels)

    def forward(self, x):
        if isinstance(x, Act):
            return self.forward_act(x)
        if self._kind() == "s2":
            raise RuntimeError("stride-2 StandardizedC2d is only reachable through Downsample")
        a, ext = _enter(x, self)
        return _exit(self.forward_act(a), ext, self)


class FP32GroupNorm(nn.GroupNorm):
    """ae.py:41-53: statistics and normalisation in fp32 regardless of the activation dtype."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)

    def forward(self, input, silu: bool = False):
        a, ext = _enter(input, self)
        y = ops.group_norm_silu(a.t, self.weight, self.bias, self.num_groups, self.eps, silu, chsums=a.stats)
        return _exit(Act(y, a.C), ext, self)

    def forward_with_skip(self, a: "Act", silu: bool = True):
        """-> (normalised activation, the input again). Consumers of the second output (the residual path) get their
        gradient summed inside the GroupNorm backward kernel (no separate accumulation pass)."""
        y, skip = ops.group_norm_silu(a.t, self.weight, self.bias, self.num_groups, self.eps, silu, with_skip=True,
                                      chsums=a.stats)
        return Act(y, a.C), Act(skip, a.C)


class AttnBlock(nn.Module):
    def __init__(self, in_channels: int):
        super().__init__()
        self.in_channels = in_channels

        self.head_dim = 64
        self.num_heads = in_channels // self.head_dim
        self.norm = FP32GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)
        self.qkv = StandardizedC2d(in_channels, in_channels * 3, kernel_size=1, bias=False)
        self.proj_out = StandardizedC2d(in_channels, in_channels, kernel_size=1, bias=False)
        nn.init.normal_(self.proj_out.weight, std=0.2 / math.sqrt(in_channels))

    def attention(self, h_) -> Act:
        a, _ = _enter(h_, self)
        return self.attention_from_normed(self.norm(a))

    def attention_from_normed(self, h: Act) -> Act:
        qkv = self.qkv.forward_act(h)  # [N,H,W,3C] : q | k | v channel blocks (ae.py:77)
        import attention as attn_core

        o = attn_core.mhsa(qkv.t, self.num_heads, self.head_dim)  # [N,H,W,C]
        return Act(o, self.in_channels)

    def forward(self, x):
        a, ext = _enter(x, self)
        hn, a_skip = self.norm.forward_with_skip(a, silu=False)
        h = self.attention_from_normed(hn)
        out = self.proj_out.forward_act(h, residual=a_skip)  # x + proj_out(attn(x)) fused in the conv epilogue
        return _exit(out, ext, self)


class ResnetBlock(nn.Module):
    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.norm1 = FP32GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)
        self.conv1 = StandardizedC2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = FP32GroupNorm(num_groups=32, num_channels=out_channels, eps=1e-6, affine=True)
        self.conv2 = StandardizedC2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            self.nin_shortcut = StandardizedC2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

        # init conv2 as very small number (ae.py:119-121)
        nn.init.normal_(self.conv2.weight, std=0.0001 / self.out_channels)
        nn.init.zeros_(self.conv2.bias)
        self.counter = 0

    def _recompute(self, a: Act) -> Act:
        """Grad-enabled path of enable_recompute: the block as one autograd node that saves only x."""
        nin = self.nin_shortcut if self.in_channels != self.out_channels else None
        spec = (self.norm1.num_groups, self.norm1.eps, self.norm2.num_groups, self.norm2.eps, self.conv1._packed,
                self.conv2._packed, nin._packed if nin is not None else None)
        out, stats = ops.resnet_block_recompute(
            a.t, a.stats, spec, self.norm1.weight, self.norm1.bias, self.conv1.weight, self.conv1.bias,
            self.norm2.weight, self.norm2.bias, self.conv2.weight, self.conv2.bias,
            nin.weight if nin is not None else None, nin.bias if nin is not None else None)
        return Act(out, self.out_channels, stats)

    def forward(self, x):
        a, ext = _enter(x, self)
        if torch.is_grad_enabled() and getattr(self, "_vqb_recompute", False):
            return _exit(self._recompute(a), ext, self)
        h, a_skip = self.norm1.forward_with_skip(a, silu=True)
        h = self.conv1.forward_act(h, want_stats=_stats_fusion())  # norm2's statistics from conv1's epilogue
        h = self.norm2(h, silu=True)
        skip = self.nin_shortcut.forward_act(a_skip) if self.in_channels != self.out_channels else a_skip
        out = self.conv2.forward_act(h, residual=skip, want_stats=_stats_fusion())  # x + h fused in the epilogue
        return _exit(out, ext, self)


def enable_recompute(module: nn.Module, enabled: bool = True) -> nn.Module:
    """Makes every ResnetBlock under `module` (encoder, decoder, the HR decoder's extra level) recompute its inner
    activations in the backward (enabled=False restores the default); returns `module`.

    With the flag set, a grad-enabled forward of a block keeps only its input (plus two [N, 32, 2] GroupNorm records)
    for the backward instead of also hn = swish(norm1(x)), h = conv1(hn) and h2 = swish(norm2(h)), and rebuilds those
    three there bit for bit: less activation memory for one extra conv1 and two GroupNorm apply passes per block in the
    backward. The forward, and the gradients, are those of the default path. No-grad forwards are unchanged."""
    for m in module.modules():
        if isinstance(m, ResnetBlock):
            m._vqb_recompute = bool(enabled)
    return module


class Downsample(nn.Module):
    def __init__(self, in_channels: int):
        super().__init__()
        self.conv = StandardizedC2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def forward(self, x):
        # F.pad(x, (0,1,0,1)) + stride-2 conv (ae.py:150-154): the pad row/column is the TMA unit's zero fill
        a, ext = _enter(x, self)
        return _exit(self.conv.forward_act(a, want_stats=_stats_fusion()), ext, self)


class Upsample(nn.Module):
    def __init__(self, in_channels: int):
        super().__init__()
        self.conv = StandardizedC2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x):
        # nearest x2 + conv3x3 as four 2x2-tap phase convs over the low-res tensor (no 4x intermediate, 4/9 of the MACs)
        a, ext = _enter(x, self)
        fuse = _stats_fusion()
        y = ops.upsample_conv(a.t, self.conv.weight, self.conv.bias, self.conv._packed, want_stats=fuse)
        if fuse:
            return _exit(Act(y[0], self.conv.out_channels, y[1]), ext, self)
        return _exit(Act(y, self.conv.out_channels), ext, self)


class Encoder(nn.Module):
    def __init__(
        self,
        resolution: int,
        in_channels: int,
        ch: int,
        ch_mult: list[int],
        num_res_blocks: int,
        z_channels: int,
        use_attn: bool = True,
        use_wavelet: bool = False,
    ):
        super().__init__()
        self.ch = ch
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.use_wavelet = use_wavelet
        if self.use_wavelet:
            self.wavelet_transform = wavelet_transform_multi_channel
            self.conv_in = StandardizedC2d(4 * in_channels, self.ch * 2, kernel_size=3, stride=1, padding=1)
            ch_mult[0] *= 2  # mutates the caller's list exactly like ae.py:194 (VAE relies on it)
        else:
            self.wavelet_transform = nn.Identity()
            self.conv_in = StandardizedC2d(in_channels, self.ch, kernel_size=3, stride=1, padding=1)

        curr_res = resolution
        in_ch_mult = (2 if self.use_wavelet else 1,) + tuple(ch_mult)
        self.in_ch_mult = in_ch_mult
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
            if i_level != self.num_resolutions - 1 and not (self.use_wavelet and i_level == 0):
                down.downsample = Downsample(block_in)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in)
        self.mid.attn_1 = AttnBlock(block_in) if use_attn else nn.Identity()
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in)
        self.norm_out = FP32GroupNorm(num_groups=32, num_channels=block_in, eps=1e-6, affine=True)
        self.conv_out = StandardizedC2d(block_in, z_channels, kernel_size=3, stride=1, padding=1)
        for module in self.modules():
            if isinstance(module, StandardizedC2d) and module.bias is not None:  # fix of ae.py:233-235 (fact 6)
                nn.init.zeros_(module.bias)
            if isinstance(module, nn.GroupNorm):
                nn.init.zeros_(module.bias)

    def forward(self, x) -> Tensor:
        _param_dtype(self)
        if self.use_wavelet and x.is_cuda and not x.requires_grad:
            # wavelet analysis (utils.py:229-247) fused with the NCHW->NHWC conversion: one kernel, no fp32 intermediate
            import utils as _u

            a = Act(ops.wavelet_to_nhwc(x, _u.filters_expanded), 4 * x.shape[1])
        else:
            h = self.wavelet_transform(x)
            fat = h.shape[1] <= 8 and ops.fat_conv_enabled()  # RGB input: 3 fat taps of 24, not 9 taps of 8 channels
            a = Act(ops.to_nhwc(h, frame=fat), h.shape[1], framed=fat)
        a = self.conv_in.forward_act(a, want_stats=_stats_fusion())
        for i_level in range(self.num_resolutions):
            for i_block in range(self.num_res_blocks):
                a = self.down[i_level].block[i_block](a)
                if len(self.down[i_level].attn) > 0:
                    a = self.down[i_level].attn[i_block](a)
            if i_level != self.num_resolutions - 1 and not (self.use_wavelet and i_level == 0):
                a = self.down[i_level].downsample(a)
        a = self.mid.block_1(a)
        if not isinstance(self.mid.attn_1, nn.Identity):
            a = self.mid.attn_1(a)
        a = self.mid.block_2(a)
        a = self.norm_out(a, silu=True)
        return self.conv_out.forward_act(a, nchw_out=True)  # [B, z, h, w] in the parameters' dtype


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
        use_attn: bool = True,
    ):
        super().__init__()
        self.ch = ch
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.ffactor = 2 ** (self.num_resolutions - 1)
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        self.conv_in = StandardizedC2d(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in)
        self.mid.attn_1 = AttnBlock(block_in) if use_attn else nn.Identity()
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
        self.norm_out = FP32GroupNorm(num_groups=32, num_channels=block_in, eps=1e-6, affine=True)
        self.conv_out = StandardizedC2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)

        # initialize all bias to zero
        for module in self.modules():
            if isinstance(module, StandardizedC2d) and module.bias is not None:
                nn.init.zeros_(module.bias)
            if isinstance(module, nn.GroupNorm):
                nn.init.zeros_(module.bias)

    def forward(self, z) -> Tensor:
        _param_dtype(self)
        a = Act(ops.to_nhwc(z), z.shape[1])
        a = self.conv_in.forward_act(a, want_stats=_stats_fusion())
        a = self.mid.block_1(a)
        if not isinstance(self.mid.attn_1, nn.Identity):
            a = self.mid.attn_1(a)
        a = self.mid.block_2(a)
        for i_level in reversed(range(self.num_resolutions)):
            for i_block in range(self.num_res_blocks + 1):
                a = self.up[i_level].block[i_block](a)
                if len(self.up[i_level].attn) > 0:
                    a = self.up[i_level].attn[i_block](a)
            if i_level != 0:
                a = self.up[i_level].upsample(a)
        a = self.norm_out(a, silu=True)
        return self.conv_out.forward_act(a, nchw_out=True)  # [B, out_ch, H, W] in the parameters' dtype


class DiagonalGaussian(nn.Module):
    def __init__(self, sample: bool = True, chunk_dim: int = 1):
        super().__init__()
        self.sample = sample
        self.chunk_dim = chunk_dim

    def forward(self, z) -> Tensor:
        mean = z
        if self.sample:
            std = 0.00
            return mean * (1 + std * torch.randn_like(mean))  # ae.py:342-348: identity that still advances the RNG
        else:
            return mean


class VAE(nn.Module):
    def __init__(
        self,
        resolution,
        in_channels,
        ch,
        out_ch,
        ch_mult,
        num_res_blocks,
        z_channels,
        use_attn,
        decoder_also_perform_hr,
        use_wavelet,
    ):
        super().__init__()
        self.encoder = Encoder(
            resolution=resolution,
            in_channels=in_channels,
            ch=ch,
            ch_mult=ch_mult,
            num_res_blocks=num_res_blocks,
            z_channels=z_channels,
            use_attn=use_attn,
            use_wavelet=use_wavelet,
        )
        self.decoder = Decoder(
            resolution=resolution,
            in_channels=in_channels,
            ch=ch,
            out_ch=out_ch,
            ch_mult=ch_mult + [4] if decoder_also_perform_hr else ch_mult,
            num_res_blocks=num_res_blocks,
            z_channels=z_channels,
            use_attn=use_attn,
        )
        self.reg = DiagonalGaussian()

    def forward(self, x) -> Tensor:
        z = self.encoder(x)
        z_s = self.reg(z)
        decz = self.decoder(z_s)
        return decz, z


AutoEncoder = VAE  # BASELINE.json's name for the same class


class VectorQuantizer(nn.Module):
    """VQ-GAN codebook bottleneck (BASELINE.json config 4). NOT in the reference (it has no codebook anywhere; SURVEY.md
    fact 1): standard VectorQuantizer semantics pinned by oracle/vq_oracle.py. Drop-in replacement for `VAE.reg`:

        z_q, loss, idx = vq(z)      # z [B, e_dim, h, w] fp32
        idx  = argmin_j ||z_i - e_j||^2 (canonical fp32 order, first index on ties; csrc/vq.cu)
        loss = beta * mean((sg[z_q] - z)^2) + mean((z_q - sg[z])^2)
        z_q  = z + sg[z_q - z]      (straight-through)
    """

    def __init__(self, n_e: int = 8192, e_dim: int = 16, beta: float = 0.25):
        super().__init__()
        self.n_e, self.e_dim, self.beta = n_e, e_dim, beta
        self.embedding = nn.Embedding(n_e, e_dim)
        self.embedding.weight.data.uniform_(-1.0 / n_e, 1.0 / n_e)

    def forward(self, z):
        B, D, H, W = z.shape
        zf = z.permute(0, 2, 3, 1).reshape(-1, D)
        idx, _, _ = ops.vq_argmin(zf, self.embedding.weight)
        zq = self.embedding(idx).view(B, H, W, D).permute(0, 3, 1, 2)
        loss = self.beta * torch.mean((zq.detach() - z) ** 2) + torch.mean((zq - z.detach()) ** 2)
        zq = z + (zq - z).detach()
        return zq, loss, idx.view(B, H, W)
