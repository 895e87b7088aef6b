"""Geometry descriptors (views + taps) for every convolution variant on the hot path.

A "plan" is a filled VqbConvDesc / VqbWgradDesc plus the tap map used to pack the OIHW fp32 master
weights into the bf16 [rows][slot][K] matrix the wgmma kernels read. Plans depend only on shapes
and are cached by the modules.

Variants (reference call sites):
  s1      : k x k stride-1 "same" conv (3x3 p1, 1x1 p0)                ae.py:105-117, VGG utils.py:95-111
  s2      : 3x3 stride-2 conv after F.pad(0,1,0,1)  (Downsample)       ae.py:143-154
  patch   : k x k stride-k non-overlapping conv (PatchD heads)         utils.py:156-185
  3-D     : 3x3x3 stride-1 / stride-2 / folded up-sampling convs of the video autoencoder (tae.py), see geom3_*
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Tuple

from native import (VqbConv3dDesc, VqbConv3dDgradDesc, VqbConvDesc, VqbTap, VqbTap3d, VqbView, VqbView3d,
                    VqbWgrad3dDesc, VqbWgradDesc, dense_view, dense_view3d)


def cpad(c: int) -> int:
    """Internal NHWC channel count: multiple of 8 (16-byte pixel rows)."""
    return (c + 7) // 8 * 8


@dataclass
class ConvGeom:
    """Views/taps of the A operand for out-grid (N, Ho, Wo); tapmap[slot] = source tap in the KHxKW kernel."""
    N: int
    Ho: int
    Wo: int
    C: int  # channels of the A tensor (padded)
    views: List[VqbView] = field(default_factory=list)
    taps: List[Tuple[int, int, int]] = field(default_factory=list)  # (view, dw, dh)
    tapmap: List[int] = field(default_factory=list)
    tapmask: List[int] = field(default_factory=list)  # folded weights: slot -> bit set of source taps (else empty)


def geom_s1(N, H, W, C, k) -> ConvGeom:
    p = (k - 1) // 2
    g = ConvGeom(N, H, W, C, [dense_view(N, H, W, C)])
    for kh in range(k):
        for kw in range(k):
            g.taps.append((0, kw - p, kh - p))
            g.tapmap.append(kh * k + kw)
    return g


def geom_s1_dgrad(N, H, W, Cout_pad, k) -> ConvGeom:
    """dgrad of a stride-1 same conv = same conv over dy with rotated taps (weights packed transposed)."""
    p = (k - 1) // 2
    g = ConvGeom(N, H, W, Cout_pad, [dense_view(N, H, W, Cout_pad)])
    for kh in range(k):
        for kw in range(k):
            # slot (kh,kw) reads dy at (h + kh - p, w + kw - p) and uses source tap (k-1-kh, k-1-kw)
            g.taps.append((0, kw - p, kh - p))
            g.tapmap.append((k - 1 - kh) * k + (k - 1 - kw))
    return g


def geom_s2(N, H, W, C) -> ConvGeom:
    """3x3 stride-2 conv over x padded by one zero row/col at bottom/right: out (H/2, W/2).
    Tap (kh,kw) reads x[2ho+kh, 2wo+kw] = parity view (kh&1, kw&1) at (ho + kh//2, wo + kw//2)."""
    assert H % 2 == 0 and W % 2 == 0, "Downsample needs even H, W"
    g = ConvGeom(N, H // 2, W // 2, C)
    for ph in range(2):
        for pw in range(2):
            g.views.append(VqbView(offset=(ph * W + pw) * C, Wv=W // 2, Hv=H // 2, Nv=N, _pad=0, sw=2 * C,
                                   sh=2 * W * C, sn=H * W * C))
    for kh in range(3):
        for kw in range(3):
            g.taps.append(((kh & 1) * 2 + (kw & 1), kw // 2, kh // 2))
            g.tapmap.append(kh * 3 + kw)
    return g


def geom_s2_dgrad_classes(N, H, W, Cout_pad):
    """dgrad of the stride-2 conv, one small conv per output parity class (ph,pw) of dx (H x W):
    dx[2a+ph, 2b+pw] = sum over taps with kh%2==ph, kw%2==pw of dy[a - (kh-ph)/2, b - (kw-pw)/2] * W[kh,kw].
    Returns [(ph, pw, ConvGeom over dy grid (N, H/2, W/2))]."""
    out = []
    Ho, Wo = H // 2, W // 2
    for ph in range(2):
        for pw in range(2):
            g = ConvGeom(N, Ho, Wo, Cout_pad, [dense_view(N, Ho, Wo, Cout_pad)])
            for kh in range(ph, 3, 2):
                for kw in range(pw, 3, 2):
                    g.taps.append((0, -((kw - pw) // 2), -((kh - ph) // 2)))
                    g.tapmap.append(kh * 3 + kw)
            out.append((ph, pw, g))
    return out


def geom_patch(N, H, W, C, k) -> ConvGeom:
    """k x k stride-k conv: out (H/k, W/k); tap (kh,kw) has its own strided view."""
    assert H % k == 0 and W % k == 0
    g = ConvGeom(N, H // k, W // k, C)
    for kh in range(k):
        for kw in range(k):
            g.views.append(VqbView(offset=(kh * W + kw) * C, Wv=W // k, Hv=H // k, Nv=N, _pad=0, sw=k * C,
                                   sh=k * W * C, sn=H * W * C))
            g.taps.append((kh * k + kw, 0, 0))
            g.tapmap.append(kh * k + kw)
    return g


# ---- nearest-2x upsample fused into the 3x3 conv (ae.py:164-167), SURVEY.md Appendix A ------------------------------
# out[2a+ph, 2b+pw] = sum_{i,j in 0..1} Wf[ph,pw][i][j] . x[a + OFF[ph][i], b + OFF[pw][j]]
# with Wf[ph,pw][i][j] = sum_{kh in SET[ph][i]} sum_{kw in SET[pw][j]} W[kh,kw]   (4/9 of the MACs, no 4x tensor)
_UP_OFF = {0: (-1, 0), 1: (0, 1)}
_UP_SET = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}


def _up_mask(ph, pw, i, j) -> int:
    m = 0
    for kh in _UP_SET[ph][i]:
        for kw in _UP_SET[pw][j]:
            m |= 1 << (kh * 3 + kw)
    return m


def geom_up_fwd(N, h, w, C, ph, pw) -> ConvGeom:
    """Phase (ph,pw) of upsample+conv3x3: a 2x2-tap conv over the LOW-RES x writing the (ph,pw) sub-grid of the output."""
    g = ConvGeom(N, h, w, C, [dense_view(N, h, w, C)])
    for i in range(2):
        for j in range(2):
            g.taps.append((0, _UP_OFF[pw][j], _UP_OFF[ph][i]))
            g.tapmask.append(_up_mask(ph, pw, i, j))
    return g


def up_dy_view(N, h, w, Cop, ph, pw) -> VqbView:
    """Parity view (ph,pw) of dy / out [N, 2h, 2w, Cop]."""
    return VqbView(offset=(ph * 2 * w + pw) * Cop, Wv=w, Hv=h, Nv=N, _pad=0, sw=2 * Cop, sh=2 * 2 * w * Cop,
                   sn=4 * h * w * Cop)


def geom_up_dgrad(N, h, w, Cop) -> ConvGeom:
    """dx[a,b] = sum over the 4 phases and 2x2 taps of dy_phase[a - dh, b - dw] . Wf^T : one 16-tap conv over the four
    parity views of dy."""
    g = ConvGeom(N, h, w, Cop)
    for ph in range(2):
        for pw in range(2):
            g.views.append(up_dy_view(N, h, w, Cop, ph, pw))
    for ph in range(2):
        for pw in range(2):
            for i in range(2):
                for j in range(2):
                    g.taps.append((ph * 2 + pw, -_UP_OFF[pw][j], -_UP_OFF[ph][i]))
                    g.tapmask.append(_up_mask(ph, pw, i, j))
    return g


# ---- first-layer "fat pixel" 3x3 conv over an 8-channel image ------------------------------------------------------
# The image lives in a zero-framed buffer [N][H+2][W+2][8]; horizontally adjacent pixels are CONTIGUOUS, so the conv
# becomes 3 taps (kh) whose K run starts at pixel (w-1) and covers the 8 pixels w-1..w+6 = 64 elements = one full
# 128-byte K chunk: columns 0..23 carry the three real taps (kw*8 + c), columns 24..63 meet ZERO weights. The run is 64
# wide (not 24) on purpose: a TMA box whose inner dimension is partly out of range is served row by row, a fully in-range
# 128-byte row in one piece.
# The buffer carries 64 elements of zeroed slack so the last rows stay inside the allocation.
FAT_K = 64


def fat_view(N, H, W) -> VqbView:
    return VqbView(offset=0, Wv=W, Hv=H + 2, Nv=N, _pad=0, sw=8, sh=(W + 2) * 8, sn=(H + 2) * (W + 2) * 8)


def geom_fat3(N, H, W, dgrad=False) -> ConvGeom:
    g = ConvGeom(N, H, W, FAT_K, [fat_view(N, H, W)])
    for kh in range(3):
        g.taps.append((0, 0, kh))
    g.tapmap = [8 - t for t in range(9)] if dgrad else list(range(9))  # 9 packed slots of 8 = 3 fat taps of 24
    return g


def framed_interior_view(N, H, W, C) -> VqbView:
    """The dense (N, H, W) grid seen inside a zero-framed [N][H+2][W+2][C] buffer."""
    return VqbView(offset=((W + 2) + 1) * C, Wv=W, Hv=H, Nv=N, _pad=0, sw=C, sh=(W + 2) * C, sn=(H + 2) * (W + 2) * C)


def conv_desc(g: ConvGeom, Cout: int, out_strides, flags=0, out_f32=False) -> VqbConvDesc:
    """out_strides = (on, oh, ow, oc) in elements."""
    d = VqbConvDesc()
    d.C, d.Cout, d.N, d.H, d.W = g.C, Cout, g.N, g.Ho, g.Wo
    d.nviews, d.ntaps, d.flags, d.out_f32 = len(g.views), len(g.taps), flags, 1 if out_f32 else 0
    d.on, d.oh, d.ow, d.oc = out_strides
    for i, v in enumerate(g.views):
        d.views[i] = v
    for i, (v, dw, dh) in enumerate(g.taps):
        d.taps[i] = VqbTap(view=v, dw=dw, dh=dh, _pad=0)
    return d


def nhwc_strides(H, W, Cs):
    return (H * W * Cs, W * Cs, Cs, 1)


def nchw_strides(C, H, W):
    return (C * H * W, W, 1, H * W)


def wgrad_desc(g: ConvGeom, Cout_pad: int, ksplit: int, dy_view=None, ld_override=0, col_offset=0) -> VqbWgradDesc:
    """x operand geometry = forward geometry g; dy is the dense (N, Ho, Wo, Cout_pad) tensor unless dy_view is given."""
    d = VqbWgradDesc()
    d.C, d.Cout, d.N, d.H, d.W = g.C, Cout_pad, g.N, g.Ho, g.Wo
    d.nviews, d.ntaps, d.ksplit = len(g.views), len(g.taps), ksplit
    d.ld_override, d.col_offset = ld_override, col_offset
    d.dy_view = dy_view if dy_view is not None else dense_view(g.N, g.Ho, g.Wo, Cout_pad)
    for i, v in enumerate(g.views):
        d.views[i] = v
    for i, (v, dw, dh) in enumerate(g.taps):
        d.taps[i] = VqbTap(view=v, dw=dw, dh=dh, _pad=0)
    return d


# ---- 3-D (video) convolutions of tae.py on NTHWC activations (vqb_conv3d_gemm) --------------------------------------
# Taps are (view, dw, dh, dt); tapmap / tapmask index the flattened 3x3x3 kernel, tap kt*9 + kh*3 + kw (OIDHW order).
@dataclass
class ConvGeom3d:
    """Views/taps of the A operand for the output grid (N, To, Ho, Wo)."""
    N: int
    To: int
    Ho: int
    Wo: int
    C: int  # channels of the A tensor (padded)
    views: List[VqbView3d] = field(default_factory=list)
    taps: List[Tuple[int, int, int, int]] = field(default_factory=list)  # (view, dw, dh, dt)
    tapmap: List[int] = field(default_factory=list)
    tapmask: List[int] = field(default_factory=list)


def geom3_s1(N, T, H, W, C) -> ConvGeom3d:
    """3x3x3 stride-1 conv, padding 1 (tae.py:66-78, :136-138, :165-167, :208-210, :233): 27 taps of one view."""
    g = ConvGeom3d(N, T, H, W, C, [dense_view3d(N, T, H, W, C)])
    for kt in range(3):
        for kh in range(3):
            for kw in range(3):
                g.taps.append((0, kw - 1, kh - 1, kt - 1))
                g.tapmap.append(kt * 9 + kh * 3 + kw)
    return g


def geom3_s2(N, T, H, W, C) -> ConvGeom3d:
    """Downsample (tae.py:96-104): F.pad(x, (0,1,0,1,0,1)) + 3x3x3 stride-2 conv, out (T/2, H/2, W/2). Tap (kt,kh,kw)
    reads x[2to+kt, 2ho+kh, 2wo+kw] = parity view (kt&1, kh&1, kw&1) at (to + kt//2, ho + kh//2, wo + kw//2); the pad
    plane is the view's zero fill."""
    assert T % 2 == 0 and H % 2 == 0 and W % 2 == 0, "Downsample needs even T, H, W"
    g = ConvGeom3d(N, T // 2, H // 2, W // 2, C)
    for pt in range(2):
        for ph in range(2):
            for pw in range(2):
                g.views.append(VqbView3d(offset=((pt * H + ph) * W + pw) * C, Wv=W // 2, Hv=H // 2, Tv=T // 2, Nv=N,
                                         sw=2 * C, sh=2 * W * C, st=2 * H * W * C, sn=T * H * W * C))
    for kt in range(3):
        for kh in range(3):
            for kw in range(3):
                g.taps.append(((kt & 1) * 4 + (kh & 1) * 2 + (kw & 1), kw // 2, kh // 2, kt // 2))
                g.tapmap.append(kt * 9 + kh * 3 + kw)
    return g


def _up_mask3(pt, ph, pw, i, j, k) -> int:
    m = 0
    for kt in _UP_SET[pt][i]:
        for kh in _UP_SET[ph][j]:
            for kw in _UP_SET[pw][k]:
                m |= 1 << (kt * 9 + kh * 3 + kw)
    return m


def geom3_up_fwd(N, t, h, w, C, pt, ph, pw) -> ConvGeom3d:
    """Phase (pt,ph,pw) of Upsample (tae.py:110-116: nearest x2 in T, H, W + 3x3x3 conv, padding 1): a 2x2x2-tap conv
    over the LOW-RES x writing the (pt,ph,pw) sub-grid of the output, with folded weights
    Wf[i][j][k] = sum over kt in SET[pt][i], kh in SET[ph][j], kw in SET[pw][k] of W[kt,kh,kw]. The eight phases do 8/27
    of the MACs of the literal form and never materialise the 8x tensor."""
    g = ConvGeom3d(N, t, h, w, C, [dense_view3d(N, t, h, w, C)])
    for i in range(2):
        for j in range(2):
            for k in range(2):
                g.taps.append((0, _UP_OFF[pw][k], _UP_OFF[ph][j], _UP_OFF[pt][i]))
                g.tapmask.append(_up_mask3(pt, ph, pw, i, j, k))
    return g


def up3_out_strides(t, h, w, Cop):
    """(on, ot, oh, ow, oc) of one phase sub-grid of the [N, 2t, 2h, 2w, Cop] output, and the element offset of phase
    (pt, ph, pw) is ((pt * 2h + ph) * 2w + pw) * Cop."""
    return (8 * t * h * w * Cop, 2 * 4 * h * w * Cop, 2 * 2 * w * Cop, 2 * Cop, 1)


def conv3d_desc(g: ConvGeom3d, Cout: int, out_strides, flags=0, out_f32=False) -> VqbConv3dDesc:
    """out_strides = (on, ot, oh, ow, oc) in elements."""
    d = VqbConv3dDesc()
    d.C, d.Cout, d.N, d.T, d.H, d.W = g.C, Cout, g.N, g.To, g.Ho, g.Wo
    d.nviews, d.ntaps, d.flags, d.out_f32 = len(g.views), len(g.taps), flags, 1 if out_f32 else 0
    d.on, d.ot, d.oh, d.ow, d.oc = out_strides
    for i, v in enumerate(g.views):
        d.views[i] = v
    for i, (v, dw, dh, dt) in enumerate(g.taps):
        d.taps[i] = VqbTap3d(view=v, dw=dw, dh=dh, dt=dt)
    return d


def ncthw_strides(C, T, H, W):
    return (C * T * H * W, H * W, W, 1, T * H * W)


def nthwc_strides(T, H, W, Cs):
    return (T * H * W * Cs, H * W * Cs, W * Cs, Cs, 1)


# ---- 3-D data / weight gradients (training, tae.enable_training) ---------------------------------------------------
def geom3_s1_dgrad(N, T, H, W, Cout_pad) -> ConvGeom3d:
    """dgrad of the 3x3x3 stride-1 conv = the same conv over dy with the 27 taps rotated (weights packed transposed)."""
    g = ConvGeom3d(N, T, H, W, Cout_pad, [dense_view3d(N, T, H, W, Cout_pad)])
    for kt in range(3):
        for kh in range(3):
            for kw in range(3):
                g.taps.append((0, kw - 1, kh - 1, kt - 1))
                g.tapmap.append(26 - (kt * 9 + kh * 3 + kw))
    return g


def geom3_s2_dgrad_classes(N, T, H, W, Cout_pad):
    """dgrad of the Downsample conv, one small conv per parity class (pt, ph, pw) of dx (T x H x W):
    dx[2a+pt, 2b+ph, 2c+pw] = sum over taps with kt%2==pt, kh%2==ph, kw%2==pw of
    dy[a - (kt-pt)/2, b - (kh-ph)/2, c - (kw-pw)/2] . W[kt,kh,kw]  (1 to 8 taps). The pad plane's gradient is never
    formed. Returns [(pt, ph, pw, ConvGeom3d over the dy grid (N, T/2, H/2, W/2))]; class (pt, ph, pw) writes the strided
    sub-grid s2_dgrad_out of dx."""
    out = []
    To, Ho, Wo = T // 2, H // 2, W // 2
    for pt in range(2):
        for ph in range(2):
            for pw in range(2):
                g = ConvGeom3d(N, To, Ho, Wo, Cout_pad, [dense_view3d(N, To, Ho, Wo, Cout_pad)])
                for kt in range(pt, 3, 2):
                    for kh in range(ph, 3, 2):
                        for kw in range(pw, 3, 2):
                            g.taps.append((0, -((kw - pw) // 2), -((kh - ph) // 2), -((kt - pt) // 2)))
                            g.tapmap.append(kt * 9 + kh * 3 + kw)
                out.append((pt, ph, pw, g))
    return out


def s2_dgrad_out(T, H, W, Cp, pt, ph, pw):
    """-> ((on, ot, oh, ow, oc), element offset) of parity class (pt, ph, pw) inside dx [N, T, H, W, Cp]."""
    return (T * H * W * Cp, 2 * H * W * Cp, 2 * W * Cp, 2 * Cp, 1), ((pt * H + ph) * W + pw) * Cp


def up3_dy_view(N, t, h, w, Cop, pt, ph, pw) -> VqbView3d:
    """Parity view (pt, ph, pw) of dy / out [N, 2t, 2h, 2w, Cop]."""
    return VqbView3d(offset=((pt * 2 * h + ph) * 2 * w + pw) * Cop, Wv=w, Hv=h, Tv=t, Nv=N, sw=2 * Cop,
                     sh=2 * 2 * w * Cop, st=2 * 4 * h * w * Cop, sn=8 * t * h * w * Cop)


def geom3_up_dgrad(N, t, h, w, Cop) -> ConvGeom3d:
    """dgrad of the folded up-sampling: dx[a,b,c] = sum over the 8 phases and their 2x2x2 taps of
    dy_phase[a - dt, b - dh, c - dw] . Wf^T, one 64-tap conv over the eight parity views of dy (the 3-D form of
    geom_up_dgrad). Needs the 64-entry tap table of VqbConv3dDgradDesc."""
    g = ConvGeom3d(N, t, h, w, Cop)
    for pt in range(2):
        for ph in range(2):
            for pw in range(2):
                g.views.append(up3_dy_view(N, t, h, w, Cop, pt, ph, pw))
    for pt in range(2):
        for ph in range(2):
            for pw in range(2):
                for i in range(2):
                    for j in range(2):
                        for k in range(2):
                            g.taps.append((pt * 4 + ph * 2 + pw, -_UP_OFF[pw][k], -_UP_OFF[ph][j], -_UP_OFF[pt][i]))
                            g.tapmask.append(_up_mask3(pt, ph, pw, i, j, k))
    return g


def conv3d_dgrad_desc(g: ConvGeom3d, Cout: int, out_strides) -> VqbConv3dDgradDesc:
    """64-tap form of conv3d_desc (no epilogue, bf16 output)."""
    d = VqbConv3dDgradDesc()
    d.C, d.Cout, d.N, d.T, d.H, d.W = g.C, Cout, g.N, g.To, g.Ho, g.Wo
    d.nviews, d.ntaps, d.flags, d.out_f32 = len(g.views), len(g.taps), 0, 0
    d.on, d.ot, d.oh, d.ow, d.oc = out_strides
    for i, v in enumerate(g.views):
        d.views[i] = v
    for i, (v, dw, dh, dt) in enumerate(g.taps):
        d.taps[i] = VqbTap3d(view=v, dw=dw, dh=dh, dt=dt)
    return d


def wgrad3d_desc(g: ConvGeom3d, Cout_pad: int, ksplit: int, dy_view=None, ld_override=0,
                 col_offset=0) -> VqbWgrad3dDesc:
    """x operand geometry = forward geometry g; dy is the dense (N, To, Ho, Wo, Cout_pad) tensor unless dy_view is
    given."""
    d = VqbWgrad3dDesc()
    d.C, d.Cout, d.N, d.T, d.H, d.W = g.C, Cout_pad, g.N, g.To, g.Ho, g.Wo
    d.nviews, d.ntaps, d.ksplit = len(g.views), len(g.taps), ksplit
    d.ld_override, d.col_offset = ld_override, col_offset
    d.dy_view = dy_view if dy_view is not None else dense_view3d(g.N, g.To, g.Ho, g.Wo, Cout_pad)
    for i, v in enumerate(g.views):
        d.views[i] = v
    for i, (v, dw, dh, dt) in enumerate(g.taps):
        d.taps[i] = VqbTap3d(view=v, dw=dw, dh=dh, dt=dt)
    return d
