"""Tiled encode / decode oracle: the tile planner, the blend weights and the blend, in float64 NumPy. TEST
INFRASTRUCTURE (see oracle/__init__.py).

PARITY UNPINNED BY THE REFERENCE: cloneofsimo/vqgan-training has no tiling. This file restates the definition of
DESIGN.md section 7 row 27. The module's factor f is its encoder downsampling 2^(num_resolutions - 1), or
decoder.ffactor. tile and overlap are per blended axis in sample units (frames, pixels), multiples of f,
0 <= overlap < tile. In latent units X, L, O are the extent, tile and overlap over f.

    plan       X <= L: one tile [0, X). Otherwise n = ceil((X - O) / (L - O)) tiles of length L starting at
               s_k = (k (X - L) + floor((n - 1) / 2)) // (n - 1)  (integers: s_0 = 0, s_{n-1} = X - L)
    grid       decode blends on the output grid (starts s_k f, length L f, ramp R = O f);
               encode blends on the latent grid (starts s_k, length L, ramp R = O)
    weights    r_k(x) = min(1, left, right), left = (x - a_k + 1/2) / R if k > 0 else 1,
               right = (b_k - x - 1/2) / R if k < n - 1 else 1, r_k = 1 for R = 0;
               w_k(x) = r_k(x) / sum_j r_j(x) over the tiles j covering x (summed in tile order), in float64; the kernel
               reads it rounded once to float32
    blend      out = sum over tiles in raster order (t, h, w) of (w_t (x) w_h (x) w_w) * module(window)
"""
from __future__ import annotations

import itertools

import numpy as np


def plan_axis(X: int, L: int, O: int):
    """-> (starts, length) in latent units."""
    if X <= L:
        return [0], X
    n = -(-(X - O) // (L - O))
    return [(k * (X - L) + (n - 1) // 2) // (n - 1) for k in range(n)], L


def ramp(starts, length: int, R: int) -> np.ndarray:
    """r_k over each tile's own window on the blended grid: float64 [n, length]."""
    n = len(starts)
    x = np.arange(length, dtype=np.float64)
    r = np.ones((n, length))
    if R == 0:
        return r
    for k in range(n):
        if k > 0:
            r[k] = np.minimum(r[k], (x + 0.5) / R)
        if k < n - 1:
            r[k] = np.minimum(r[k], (length - x - 0.5) / R)
    return r


def axis_weights(starts, length: int, R: int) -> np.ndarray:
    """w_k over each tile's window on the blended grid: float64 [n, length]."""
    n = len(starts)
    r = ramp(starts, length, R)
    extent = starts[-1] + length
    total = np.zeros(extent)
    for j in range(n):
        total[starts[j]:starts[j] + length] += r[j]
    return np.stack([r[k] / total[starts[k]:starts[k] + length] for k in range(n)])


def axis(X: int, tile: int, overlap: int, f: int, decode: bool):
    """One blended axis: X the latent extent, tile / overlap in sample units. -> dict with the latent plan (starts,
    length), the blended grid (gstarts, glen, gextent, R) and the float64 weights [n, glen]."""
    starts, length = plan_axis(X, tile // f, overlap // f)
    s = f if decode else 1
    gstarts, glen, R = [v * s for v in starts], length * s, overlap if decode else overlap // f
    return dict(starts=starts, length=length, gstarts=gstarts, glen=glen, gextent=X * s, R=R,
                weights=axis_weights(gstarts, glen, R))


def blend(outputs, axes) -> np.ndarray:
    """outputs: {(k_t, k_h, k_w): module output on that window, [N, C, *glen]} for every raster index of the plan;
    axes: the per-axis dicts of axis() (two for images, three for clips). -> float64 [N, C, *gextent]."""
    first = next(iter(outputs.values()))
    out = np.zeros(first.shape[:2] + tuple(a["gextent"] for a in axes))
    for idx in itertools.product(*(range(len(a["gstarts"])) for a in axes)):
        w = np.ones(())
        for a, k in zip(axes, idx):
            w = np.multiply.outer(w, a["weights"][k])
        sl = tuple(slice(a["gstarts"][k], a["gstarts"][k] + a["glen"]) for a, k in zip(axes, idx))
        out[(slice(None), slice(None)) + sl] += w * np.asarray(outputs[idx], dtype=np.float64)
    return out
