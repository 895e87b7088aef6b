"""Reconstruction-metric oracle: PSNR and SSIM per item. TEST INFRASTRUCTURE (see oracle/__init__.py).

PARITY UNPINNED BY THE REFERENCE: cloneofsimo/vqgan-training reports no reconstruction metric. This file restates the
definition of DESIGN.md section 7 row 25 (Wang et al. 2004, as in their ssim_index.m: no padding, no downsampling) in
NumPy. The value-range map is done in float32, exactly as the kernel does it; everything after it is float64.

    u      = fmin(fmax((v - lo) * inv, 0), 1)        float32, inv = 1 / (hi - lo) rounded once to float32
    PSNR   = 10 log10(1 / mean (u_x - u_y)^2)        over the item's C*H*W values; +inf when the mean is 0
    g_i    ∝ exp(-(i - 5)^2 / (2 * 1.5^2)), i = 0..10, sum 1;  w_ij = g_i g_j
    mu_x   = sum w u_x,  s_xx = sum w u_x^2 - mu_x^2,  s_xy = sum w u_x u_y - mu_x mu_y   at each valid position
    SSIM   = (2 mu_x mu_y + C1)(2 s_xy + C2) / ((mu_x^2 + mu_y^2 + C1)(s_xx + s_yy + C2)),  C1 = 0.01^2, C2 = 0.03^2,
             averaged over channels and the (H - 10)(W - 10) valid positions

An item is an image b of [B, C, H, W] or a frame (b, t) of [B, C, T, H, W]; results are [B] or [B, T].
"""
from __future__ import annotations

import numpy as np

C1 = 0.01 ** 2
C2 = 0.03 ** 2
SIGMA = 1.5
RADIUS = 5


def gaussian_1d() -> np.ndarray:
    i = np.arange(2 * RADIUS + 1, dtype=np.float64)
    g = np.exp(-(i - RADIUS) ** 2 / (2 * SIGMA ** 2))
    return g / g.sum()


def window() -> np.ndarray:
    """The 11 x 11 window w_ij = g_i g_j (float64)."""
    g = gaussian_1d()
    return np.outer(g, g)


def to_unit(v, value_range=(0.0, 1.0)) -> np.ndarray:
    """The float32 map of the definition (fmin / fmax: a NaN maps to 0, as in C)."""
    lo, hi = np.float32(value_range[0]), np.float32(value_range[1])
    inv = np.float32(1.0 / (np.float64(hi) - np.float64(lo)))
    v = np.asarray(v, dtype=np.float32)
    return np.fmin(np.fmax((v - lo) * inv, np.float32(0)), np.float32(1)).astype(np.float32)


def valid_filter(a: np.ndarray) -> np.ndarray:
    """sum_ij w_ij a[..., p + i, q + j] at every valid position (p, q) of the last two axes, float64."""
    a = np.asarray(a, dtype=np.float64)
    g = gaussian_1d()
    n = 2 * RADIUS + 1
    H, W = a.shape[-2:]
    h = sum(g[j] * a[..., :, j:j + W - n + 1] for j in range(n))
    return sum(g[i] * h[..., i:i + H - n + 1, :] for i in range(n))


def _items(u: np.ndarray) -> np.ndarray:
    """[B, C, H, W] -> [B, 1, C, H, W]; [B, C, T, H, W] -> [B, T, C, H, W] (items first, then the item's planes)."""
    return u[:, None] if u.ndim == 4 else np.moveaxis(u, 2, 1)


def moments(ux: np.ndarray, uy: np.ndarray):
    """float64 (mu_x, mu_y, s_xx, s_yy, s_xy) at every valid position of every plane of the mapped inputs."""
    ux, uy = np.asarray(ux, dtype=np.float64), np.asarray(uy, dtype=np.float64)
    mx, my = valid_filter(ux), valid_filter(uy)
    return (mx, my, valid_filter(ux * ux) - mx * mx, valid_filter(uy * uy) - my * my,
            valid_filter(ux * uy) - mx * my)


def ssim_formula(mx, my, sxx, syy, sxy):
    return (2 * mx * my + C1) * (2 * sxy + C2) / ((mx * mx + my * my + C1) * (sxx + syy + C2))


def psnr_ssim(x, y, value_range=(0.0, 1.0)):
    """-> (psnr, ssim) float64, [B] for images, [B, T] for clips."""
    x, y = np.asarray(x), np.asarray(y)
    if x.shape != y.shape or x.ndim not in (4, 5):
        raise ValueError(f"expected two [B, C, H, W] or [B, C, T, H, W] arrays of one shape, got {x.shape}, {y.shape}")
    ux, uy = _items(to_unit(x, value_range)), _items(to_unit(y, value_range))
    d = ux.astype(np.float64) - uy.astype(np.float64)
    mse = (d * d).mean(axis=(2, 3, 4))
    with np.errstate(divide="ignore"):
        psnr = 10 * np.log10(1 / mse)
    ssim = ssim_formula(*moments(ux, uy)).mean(axis=(2, 3, 4))
    if x.ndim == 4:
        return psnr[:, 0], ssim[:, 0]
    return psnr, ssim


def psnr_ssim_torch(x, y, value_range=(0.0, 1.0), dtype=None):
    """The same definition in PyTorch on x's device: the float32 map, then grouped F.conv2d with the separable window in
    `dtype` (default float64). -> (psnr, ssim) in `dtype`, [B] or [B, T]. The float64 form cross-checks the kernel on
    the GPU; the float32 form is the eager cuDNN peer of tools/metrics_bench.py."""
    import torch
    import torch.nn.functional as F

    dtype = dtype or torch.float64
    lo, hi = np.float32(value_range[0]), np.float32(value_range[1])
    inv = float(np.float32(1.0 / (np.float64(hi) - np.float64(lo))))

    def unit(v):
        v = v if v.dim() == 5 else v.unsqueeze(2)
        v = v.transpose(1, 2).reshape(-1, *v.shape[-2:]).float()  # [B*T*C, H, W]: items' planes in (b, t, c) order
        return ((v - float(lo)) * inv).clamp(0, 1).to(dtype).unsqueeze(1)

    B = x.shape[0]
    T = x.shape[2] if x.dim() == 5 else 1
    ux, uy = unit(x), unit(y)
    g = torch.tensor(gaussian_1d(), dtype=dtype, device=x.device)

    def filt(a):
        return F.conv2d(F.conv2d(a, g.view(1, 1, 1, -1)), g.view(1, 1, -1, 1))

    mse = (ux - uy).pow(2).reshape(B * T, -1).mean(1)
    mx, my = filt(ux), filt(uy)
    s = ssim_formula(mx, my, filt(ux * ux) - mx * mx, filt(uy * uy) - my * my, filt(ux * uy) - mx * my)
    psnr, ssim = 10 * torch.log10(1 / mse), s.reshape(B * T, -1).mean(1)
    shape = (B,) if x.dim() == 4 else (B, T)
    return psnr.view(shape), ssim.view(shape)
