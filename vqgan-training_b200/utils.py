"""H100-native drop-in for the reference `utils.py`: LPIPS, ScalingLayer, NetLinLayer, vgg16, PatchDiscriminator,
normalize_tensor, spatial_average, and the wavelet front-end — same class names, constructor signatures and
state_dict keys (utils.py:8-247), with the VGG16 trunks, LPIPS tail and discriminator heads running on the sm_90a
kernels of libvqb200.so:

  13 VGG conv3x3 + bias + ReLU        -> wgmma implicit-GEMM conv with fused bias/ReLU epilogue (csrc/conv_gemm.cu);
                                         the data-gradient epilogue applies the ReLU gate of the producing layer
  4 max-pools                         -> csrc/lpips.cu (backward fuses the ReLU gate)
  LPIPS tail (normalise, diff^2, lin, spatial mean, 5-way sum; ~12 ATen kernels per layer in the reference)
                                      -> one kernel per layer and direction (csrc/lpips.cu)
  PatchD heads k4s4 / k2s2 / k1       -> the same conv kernel with one strided TMA view per filter tap

Offline note: the reference downloads torchvision's ImageNet VGG16 weights and `vgg.pth`; when neither is reachable
(no network) the constructors keep torchvision's random initialisation and warn instead of crashing, so that
seeded-weight parity tests and benchmarks run anywhere. Numerics of the *pretrained* metric are therefore unpinned
(SURVEY.md §8c).
"""
from __future__ import annotations

import os
import sys
import warnings
from collections import OrderedDict, namedtuple

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import torch
import torch.nn as nn
from torchvision import models

import ops


def _offline() -> bool:
    """VQB_OFFLINE=1 is the explicit opt-in (tests, benchmarks, smoke) to run with random-initialised VGG16 / LPIPS lin
    weights. Without it a missing pretrained file is an ERROR: silently training against a random perceptual metric
    (whose uniform(-b, b) lin weights can be driven down by *increasing* feature differences) is never what a run wants."""
    return os.environ.get("VQB_OFFLINE", "0") == "1"


def _torchvision_vgg16_features(pretrained: bool):
    """utils.py:95,148 call models.vgg16(pretrained=True); keep that call (so the usual monkey-patches apply)."""
    if _offline():  # never touch the network
        return models.vgg16(weights=None).features
    try:
        return models.vgg16(pretrained=pretrained).features
    except Exception as e:  # URLError etc.
        raise RuntimeError(f"torchvision VGG16 ImageNet weights unavailable ({type(e).__name__}: {e}). Provide them in "
                           "the torch hub cache, or set VQB_OFFLINE=1 to run with random-initialised VGG16 weights "
                           "(tests / benchmarks only)") from e


VGG_LPIPS_URL = "https://heibox.uni-heidelberg.de/seafhttp/files/9535cbee-6558-4c0c-8743-78f5e56ea75e/vgg.pth"


def broadcast_module_state(module: nn.Module, src: int = 0):
    """Frozen modules (LPIPS and its VGG trunk) are not DDP-wrapped: make every rank use rank `src`'s weights, so that a
    per-rank difference in what could be loaded can never make ranks optimise different objectives."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return
    for t in list(module.parameters()) + list(module.buffers()):
        dist.broadcast(t.data, src)
    if any(p.is_cuda for p in module.parameters()):
        ops.weights_updated(list(module.parameters()))


def _as_b200_conv(layer: nn.Conv2d):
    """Wraps a torchvision conv's Parameters into a wgmma-backed StandardizedC2d without consuming RNG."""
    from ae import StandardizedC2d

    with torch.random.fork_rng(devices=[]):
        c = StandardizedC2d(layer.in_channels, layer.out_channels, kernel_size=layer.kernel_size,
                            stride=layer.stride, padding=layer.padding)
    c.weight = layer.weight
    c.bias = layer.bias
    return c


def _convert_features(feats):
    out = []
    for layer in feats:
        out.append(_as_b200_conv(layer) if isinstance(layer, nn.Conv2d) else layer)
    return out


def _run_trunk_slice(seq, a, first_input_is_relu):
    """seq: modules of one VGG slice (MaxPool2d / conv / ReLU placeholders). Fused: conv+bias+ReLU, pool."""
    from ae import Act

    prev_relu = first_input_is_relu
    for m in seq:
        if isinstance(m, nn.MaxPool2d):
            a = Act(ops.maxpool2(a.t), a.C)
            prev_relu = False  # the pool backward already gates by the pre-pool activation
        elif isinstance(m, nn.Conv2d):
            a = m.forward_act(a, relu=True, input_is_relu=prev_relu)
            prev_relu = True
        # nn.ReLU placeholders are fused into the conv epilogue
    return a


class LPIPS(nn.Module):
    # Learned perceptual metric
    def __init__(self, use_dropout=True):
        super().__init__()
        self.scaling_layer = ScalingLayer()
        self.chns = [64, 128, 256, 512, 512]  # vg16 features
        self.net = vgg16(pretrained=True, requires_grad=False)
        self.lin0 = NetLinLayer(self.chns[0], use_dropout=use_dropout)
        self.lin1 = NetLinLayer(self.chns[1], use_dropout=use_dropout)
        self.lin2 = NetLinLayer(self.chns[2], use_dropout=use_dropout)
        self.lin3 = NetLinLayer(self.chns[3], use_dropout=use_dropout)
        self.lin4 = NetLinLayer(self.chns[4], use_dropout=use_dropout)
        self.load_from_pretrained()
        for param in self.parameters():
            param.requires_grad = False
        self.dropout_seeds = None       # test hook: five fixed per-layer seeds for the train-mode dropout masks
        self.last_dropout_seeds = None

    def load_from_pretrained(self, name="vgg_lpips"):
        """utils.py:25-37: ./vgg.pth, else download it (same URL), else fail — unless VQB_OFFLINE=1."""
        if _offline() and not os.path.exists("vgg.pth"):
            return
        try:
            data = torch.load("vgg.pth", map_location=torch.device("cpu"))
        except Exception:
            print("Failed to load vgg.pth, downloading...")
            try:
                import urllib.request

                urllib.request.urlretrieve(VGG_LPIPS_URL, "vgg.pth")
                data = torch.load("vgg.pth", map_location=torch.device("cpu"))
            except Exception as e:
                raise RuntimeError(f"vgg.pth (LPIPS linear weights) is missing and could not be downloaded ({e}); place "
                                   "it in the working directory, or set VQB_OFFLINE=1 to run with random lin layers "
                                   "(tests / benchmarks only)") from e
        self.load_state_dict(data, strict=False)

    def forward(self, input, target, *, frames=None):
        """input, target: [B, 3, H, W] images -> [B, 1, 1, 1]; or [B, 3, T, H, W] clips -> [B*T', 1, 1, 1], the metric of
        every selected frame, frames folded into the batch in (b, t) order. frames: optional [B, T'] integer tensor or
        list of distinct frames per clip (default: every frame, T' = T)."""
        from ae import Act

        clip = _clip_selection(input, frames, target)
        # SURVEY.md fact 5: the reference never calls .eval() on LPIPS, so its nn.Dropout(0.5) in front of every lin layer
        # is live during training. Honoured here: in train mode (and when the lin layer has a Dropout) the fused tail
        # applies a counter-based keep mask; the per-call seed comes from torch's CPU generator (torch.manual_seed
        # reproducible, no device sync). `dropout_seeds` (test hook) pins the five per-layer seeds.
        fat = ops.fat_conv_enabled()
        a0 = Act(self.scaling_layer.to_act(input, fat, clip), 3, framed=fat)
        with torch.no_grad():
            a1 = Act(self.scaling_layer.to_act(target, fat, clip), 3, framed=fat)
            outs1 = self.net.forward_acts(a1)
        outs0 = self.net.forward_acts(a0)
        lins = [self.lin0, self.lin1, self.lin2, self.lin3, self.lin4]
        val = None
        seeds = [None] * 5
        if self.training and any(isinstance(m, nn.Dropout) and m.p > 0 for m in self.lin0.model):
            seeds = self.dropout_seeds
            if seeds is None:
                seeds = [int(v) for v in torch.randint(0, 2 ** 62, (5,), dtype=torch.int64)]
            self.last_dropout_seeds = list(seeds)
        for kk in range(len(self.chns)):
            r = ops.lpips_tail(outs0[kk].t, outs1[kk].t, lins[kk].model[-1].weight, seeds[kk])
            val = r if val is None else val + r
        return val.reshape(-1, 1, 1, 1)


class ScalingLayer(nn.Module):
    def __init__(self):
        super(ScalingLayer, self).__init__()
        self.register_buffer("shift", torch.Tensor([-0.030, -0.088, -0.188])[None, :, None, None])
        self.register_buffer("scale", torch.Tensor([0.458, 0.448, 0.450])[None, :, None, None])

    def forward(self, inp):
        return (inp - self.shift) / self.scale

    def to_act(self, inp, frame=False, clip=None):
        """(inp - shift) / scale fused into the NCHW fp32 -> NHWC bf16 layout kernel (optionally zero-framed for the
        fat-pixel first VGG conv). clip: the checked (selection, T') of _clip_selection for a [B, 3, T, H, W] clip,
        whose selected frames become the batch (ops.ClipToFrames)."""
        shift = self.shift.reshape(-1).float().contiguous()
        inv = (1.0 / self.scale.reshape(-1).float()).contiguous()
        if clip is not None:
            return ops.ClipToFrames.apply(inp, shift, inv, frame, *clip)
        return ops.to_nhwc(inp, shift, inv, frame)


def _clip_selection(x, frames, target=None):
    """Checks a call of LPIPS / PatchDiscriminator before anything is launched. A 4-D image batch -> None (the image
    path). A [B, 3, T, H, W] clip (and a target of the same shape) -> (int32 CPU selection or None, T') from
    ops.clip_frame_selection."""
    if x.dim() != 5:
        if frames is not None:
            raise ValueError(f"frames= selects frames of [B, 3, T, H, W] clips; the input has shape {tuple(x.shape)}")
        if target is not None and target.dim() == 5:
            raise ValueError(f"target shape {tuple(target.shape)} differs from input shape {tuple(x.shape)}")
        return None
    if x.shape[1] != 3:
        raise ValueError(f"expected a [B, 3, T, H, W] clip, got {x.shape[1]} channels (shape {tuple(x.shape)})")
    if target is not None and tuple(target.shape) != tuple(x.shape):
        raise ValueError(f"target shape {tuple(target.shape)} differs from input shape {tuple(x.shape)}")
    return ops.clip_frame_selection(frames, x.shape[0], x.shape[2])


class NetLinLayer(nn.Module):
    """A single linear layer which does a 1x1 conv"""

    def __init__(self, chn_in, chn_out=1, use_dropout=False):
        super(NetLinLayer, self).__init__()
        layers = [nn.Dropout()] if (use_dropout) else []
        layers += [nn.Conv2d(chn_in, chn_out, 1, stride=1, padding=0, bias=False)]
        self.model = nn.Sequential(*layers)


class vgg16(torch.nn.Module):
    def __init__(self, requires_grad=False, pretrained=True):
        super(vgg16, self).__init__()
        vgg_pretrained_features = _convert_features(_torchvision_vgg16_features(pretrained))
        self.slice1 = torch.nn.Sequential()
        self.slice2 = torch.nn.Sequential()
        self.slice3 = torch.nn.Sequential()
        self.slice4 = torch.nn.Sequential()
        self.slice5 = torch.nn.Sequential()
        self.N_slices = 5
        for x in range(4):
            self.slice1.add_module(str(x), vgg_pretrained_features[x])
        for x in range(4, 9):
            self.slice2.add_module(str(x), vgg_pretrained_features[x])
        for x in range(9, 16):
            self.slice3.add_module(str(x), vgg_pretrained_features[x])
        for x in range(16, 23):
            self.slice4.add_module(str(x), vgg_pretrained_features[x])
        for x in range(23, 30):
            self.slice5.add_module(str(x), vgg_pretrained_features[x])
        if not requires_grad:
            for param in self.parameters():
                param.requires_grad = False

    def forward_acts(self, a):
        outs = []
        for i, s in enumerate([self.slice1, self.slice2, self.slice3, self.slice4, self.slice5]):
            a = _run_trunk_slice(s, a, first_input_is_relu=False)
            outs.append(a)
        return outs

    def forward(self, X):
        from ae import Act

        outs = self.forward_acts(Act(ops.to_nhwc(X), X.shape[1]))
        vgg_outputs = namedtuple("VggOutputs", ["relu1_2", "relu2_2", "relu3_3", "relu4_3", "relu5_3"])
        return vgg_outputs(*[ops.to_nchw(o.t, o.C) for o in outs])


def normalize_tensor(x, eps=1e-10):
    norm_factor = torch.sqrt(torch.sum(x**2, dim=1, keepdim=True))
    return x / (norm_factor + eps)


def spatial_average(x, keepdim=True):
    return x.mean([2, 3], keepdim=keepdim)


class PatchDiscriminator(nn.Module):
    def __init__(self):
        super(PatchDiscriminator, self).__init__()
        from ae import StandardizedC2d

        self.scaling_layer = ScalingLayer()

        feats = _convert_features(_torchvision_vgg16_features(True))

        def sl(a, b):  # slicing a Sequential keeps the original module names -> keys slice{k}.0.{torchvision idx}
            return nn.Sequential(nn.Sequential(OrderedDict((str(i), feats[i]) for i in range(a, b))))

        self.slice1 = sl(0, 4)
        self.slice2 = sl(4, 9)
        self.slice3 = sl(9, 16)
        self.slice4 = sl(16, 23)
        self.slice5 = sl(23, 30)

        self.binary_classifier1 = nn.Sequential(
            StandardizedC2d(64, 32, kernel_size=4, stride=4, padding=0, bias=True),
            nn.ReLU(),
            StandardizedC2d(32, 1, kernel_size=4, stride=4, padding=0, bias=True),
        )
        nn.init.zeros_(self.binary_classifier1[-1].weight)

        self.binary_classifier2 = nn.Sequential(
            StandardizedC2d(128, 64, kernel_size=4, stride=4, padding=0, bias=True),
            nn.ReLU(),
            StandardizedC2d(64, 1, kernel_size=2, stride=2, padding=0, bias=True),
        )
        nn.init.zeros_(self.binary_classifier2[-1].weight)

        self.binary_classifier3 = nn.Sequential(
            StandardizedC2d(256, 128, kernel_size=2, stride=2, padding=0, bias=True),
            nn.ReLU(),
            StandardizedC2d(128, 1, kernel_size=2, stride=2, padding=0, bias=True),
        )
        nn.init.zeros_(self.binary_classifier3[-1].weight)

        self.binary_classifier4 = nn.Sequential(
            StandardizedC2d(512, 1, kernel_size=2, stride=2, padding=0, bias=True),
        )
        nn.init.zeros_(self.binary_classifier4[-1].weight)

        self.binary_classifier5 = nn.Sequential(
            StandardizedC2d(512, 1, kernel_size=1, stride=1, padding=0, bias=True),
        )
        nn.init.zeros_(self.binary_classifier5[-1].weight)

    @staticmethod
    def _head(seq, feat):
        """conv (+ReLU, conv): every head reads a post-ReLU activation -> its data gradient is ReLU-gated."""
        if len(seq) == 3:
            h = seq[0].forward_act(feat, relu=True, input_is_relu=True)
            return seq[2].forward_act(h, input_is_relu=True, nchw_out=True)
        return seq[0].forward_act(feat, input_is_relu=True, nchw_out=True)

    def forward(self, x, *, frames=None):
        """x: [B, 3, H, W] images -> logits [B, (H/16)(W/16)]; or a [B, 3, T, H, W] clip -> [B*T', (H/16)(W/16)], the
        logits of every selected frame, frames folded into the batch in (b, t) order (frames as in LPIPS.forward)."""
        from ae import Act

        clip = _clip_selection(x, frames)
        fat = ops.fat_conv_enabled()
        a = Act(self.scaling_layer.to_act(x, fat, clip), 3, framed=fat)
        f1 = _run_trunk_slice(self.slice1[0], a, False)
        f2 = _run_trunk_slice(self.slice2[0], f1, False)
        f3 = _run_trunk_slice(self.slice3[0], f2, False)
        f4 = _run_trunk_slice(self.slice4[0], f3, False)
        f5 = _run_trunk_slice(self.slice5[0], f4, False)

        bc1 = self._head(self.binary_classifier1, f1).flatten(1)
        bc2 = self._head(self.binary_classifier2, f2).flatten(1)
        bc3 = self._head(self.binary_classifier3, f3).flatten(1)
        bc4 = self._head(self.binary_classifier4, f4).flatten(1)
        bc5 = self._head(self.binary_classifier5, f5).flatten(1)

        return bc1 + bc2 + bc3 + bc4 + bc5


dec_lo, dec_hi = (
    torch.Tensor([-0.1768, 0.3536, 1.0607, 0.3536, -0.1768, 0.0000]),
    torch.Tensor([0.0000, -0.0000, 0.3536, -0.7071, 0.3536, -0.0000]),
)

filters = torch.stack(
    [
        dec_lo.unsqueeze(0) * dec_lo.unsqueeze(1),
        dec_lo.unsqueeze(0) * dec_hi.unsqueeze(1),
        dec_hi.unsqueeze(0) * dec_lo.unsqueeze(1),
        dec_hi.unsqueeze(0) * dec_hi.unsqueeze(1),
    ],
    dim=0,
)

filters_expanded = filters.unsqueeze(1)


def prepare_filter(device):
    global filters_expanded
    filters_expanded = filters_expanded.to(device)


def wavelet_transform_multi_channel(x, levels=4):
    """utils.py:229-247. Fixed 6x6 analysis filters, stride 2 after pad 2 -> [B, 4C, H/2, W/2]; `levels` is unused in
    the reference too. Input-side op outside BASELINE's configs (SURVEY.md §8f item 3): runs as a grouped ATen conv."""
    B, C, H, W = x.shape
    padded = torch.nn.functional.pad(x, (2, 2, 2, 2))
    w = filters_expanded.to(device=x.device, dtype=x.dtype).repeat(C, 1, 1, 1)  # [(c,band),1,6,6]
    res = torch.nn.functional.conv2d(padded, w, stride=2, groups=C)
    return res


def test_patch_discriminator():
    vggDiscriminator = PatchDiscriminator().cuda()
    x = vggDiscriminator(torch.randn(1, 3, 256, 256).cuda())
    print(x.shape)


if __name__ == "__main__":
    test_patch_discriminator()
