"""Tiled encode / decode: run an autoencoder's encoder or decoder over overlapping windows of an input too large for one
pass, and blend the windows' outputs into the full result on the native `vqb_tile_blend` kernel (DESIGN.md section
3.11, definition in section 7 row 27).

    tiling.encode(encoder, x, tile=..., overlap=...)   x [B, C, T, H, W] (tae) or [B, C, H, W] (ae) -> encoder output
    tiling.decode(decoder, z, tile=..., overlap=...)   z latents -> decoder output

`tile` and `overlap` are given per blended axis in sample units: (T, H, W) for clips, (H, W) for images. Each must be a
multiple of the module's factor f (the encoder's downsampling 2^(num_resolutions - 1), or `decoder.ffactor`) with
0 <= overlap < tile. Each window runs through the module's own forward, so peak memory follows the tile's size, not the
input's. Tiled output is not the untiled output: GroupNorm statistics and the mid-block attention see one window at a
time. When every axis fits in one tile the module is called once on the whole input and its output returned as is.
"""
from __future__ import annotations

import itertools

import torch
from torch import nn

import ae
import native
import ops
import tae


def plan_axis(X: int, L: int, O: int):
    """Tiles over one axis in latent units: X extent, L tile, O overlap (0 <= O < L). -> (starts, length). One tile
    [0, X) when X <= L; otherwise the fewest tiles of length L whose stride is at most L - O, spread evenly so that the
    first starts at 0 and the last ends at X."""
    if X <= L:
        return [0], X
    n = -(-(X - O) // (L - O))
    return [(k * (X - L) + (n - 1) // 2) // (n - 1) for k in range(n)], L


def axis_weights(starts, length: int, R: int) -> torch.Tensor:
    """Blend weights of each tile over its own window of the blended grid: float64 [n, length]. A tile's ramp rises
    over R cells from each side it shares with a neighbour, r = min(1, (x + 1/2) / R, (length - x - 1/2) / R); the
    weights are the ramps normalised by their sum over the tiles covering each cell (summed in tile order)."""
    n = len(starts)
    x = torch.arange(length, dtype=torch.float64)
    r = torch.ones(n, length, dtype=torch.float64)
    if R > 0:
        for k in range(n):
            if k > 0:
                r[k] = torch.minimum(r[k], (x + 0.5) / R)
            if k < n - 1:
                r[k] = torch.minimum(r[k], (length - x - 0.5) / R)
    total = torch.zeros(starts[-1] + length, dtype=torch.float64)
    for j in range(n):
        total[starts[j]:starts[j] + length] += r[j]
    return torch.stack([r[k] / total[starts[k]:starts[k] + length] for k in range(n)])


class _Axis:
    """One blended axis: the latent plan and the blended grid (the output grid for decode, the latent grid for
    encode), with the fp32 weight table [n, glen] the kernel reads."""

    def __init__(self, X: int, tile: int, overlap: int, f: int, decode: bool):
        self.starts, self.length = plan_axis(X, tile // f, overlap // f)
        s = f if decode else 1
        self.gstarts = [v * s for v in self.starts]
        self.glen, self.gextent = self.length * s, X * s
        self.table = axis_weights(self.gstarts, self.glen, overlap if decode else overlap // f).float()

    @property
    def n(self):
        return len(self.starts)

    def prev_end(self, k):
        return self.gstarts[k - 1] + self.glen if k > 0 else self.gstarts[k]

    def next_start(self, k):
        return self.gstarts[k + 1] if k < self.n - 1 else self.gextent


_MODULES = {tae.Encoder: (5, False), tae.Decoder: (5, True), ae.Encoder: (4, False), ae.Decoder: (4, True)}


def factor(module: nn.Module) -> int:
    """The module's factor f between sample and latent extents."""
    if isinstance(module, (tae.Decoder, ae.Decoder)):
        return module.ffactor
    return 2 ** (module.num_resolutions - 1)


def _axes(module, x, tile, overlap, decode):
    """Validates the call (before anything launches) and plans every blended axis."""
    kind = next((v for k, v in _MODULES.items() if isinstance(module, k)), None)
    what = "decode" if decode else "encode"
    if kind is None or kind[1] != decode:
        want = "tae.Decoder or ae.Decoder" if decode else "tae.Encoder or ae.Encoder"
        raise TypeError(f"tiling.{what}: expected a {want}, got {type(module).__name__}")
    rank = kind[0]
    f = factor(module)
    if not isinstance(x, torch.Tensor) or x.dim() != rank:
        shape = tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
        raise ValueError(f"tiling.{what}: {type(module).__module__}.{type(module).__name__} takes a {rank}-D input, "
                         f"got {shape} (f = {f})")
    nax = rank - 2
    ext = tuple(x.shape[2:])
    for name, v in (("tile", tile), ("overlap", overlap)):
        if not (isinstance(v, (tuple, list)) and len(v) == nax and all(isinstance(e, int) for e in v)):
            raise ValueError(f"tiling.{what}: {name} must be {nax} integers in sample units "
                             f"({'(T, H, W)' if nax == 3 else '(H, W)'}), got {v!r} (f = {f}, input {tuple(x.shape)})")
    for L, O in zip(tile, overlap):
        if L <= 0 or O < 0 or L % f or O % f:
            raise ValueError(f"tiling.{what}: tile {tuple(tile)} and overlap {tuple(overlap)} must be non-negative "
                             f"multiples of f = {f} with tile > 0 (input {tuple(x.shape)})")
        if O >= L:
            raise ValueError(f"tiling.{what}: overlap {tuple(overlap)} must be smaller than tile {tuple(tile)} on "
                             f"every axis (f = {f}, input {tuple(x.shape)})")
    if min(x.shape) <= 0 or (not decode and any(e % f for e in ext)):
        raise ValueError(f"tiling.{what}: the input's extents must be positive{'' if decode else ' multiples of f'} "
                         f"(f = {f}), got {tuple(x.shape)}")
    if x.requires_grad:
        raise RuntimeError(f"tiling.{what} runs inference only: the input requires grad; pass a detached tensor")
    if torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters()):
        raise RuntimeError(f"tiling.{what} runs inference only: call it under torch.no_grad() (or "
                           "torch.inference_mode()), or freeze the module's parameters")
    ops.require_cuda(x)
    X = ext if decode else tuple(e // f for e in ext)
    return [_Axis(Xa, L, O, f, decode) for Xa, L, O in zip(X, tile, overlap)], f


def _run(module, x, tile, overlap, decode):
    axes, f = _axes(module, x, tile, overlap, decode)
    if all(a.n == 1 for a in axes):
        return module(x)
    s = 1 if decode else f  # input units per latent unit
    grid_axes = [_Axis(1, 1, 0, 1, True)] * (3 - len(axes)) + axes  # an image blends as a clip of one frame
    tables = [a.table.to(x.device) for a in grid_axes]
    acc = out = None
    for idx in itertools.product(*(range(a.n) for a in axes)):
        window = tuple(slice(a.starts[k] * s, (a.starts[k] + a.length) * s) for a, k in zip(axes, idx))
        y = module(x[(slice(None), slice(None)) + window].contiguous()).contiguous()
        if acc is None:
            grid = tuple(y.shape[:2]) + tuple(a.gextent for a in axes)
            acc = torch.empty(grid, device=x.device, dtype=torch.float32)
            out = torch.empty(grid, device=x.device, dtype=y.dtype) if y.dtype == torch.bfloat16 else acc
        want = tuple(acc.shape[:2]) + tuple(a.glen for a in axes)
        if tuple(y.shape) != want:
            raise RuntimeError(f"tiling: the module returned {tuple(y.shape)} for a window, expected {want}")
        k3 = (0,) * (3 - len(axes)) + idx
        native.check(ops._L().vqb_tile_blend(
            y.data_ptr(), int(y.dtype == torch.bfloat16), acc.data_ptr(), None if out is acc else out.data_ptr(),
            *acc.shape[:2], *(a.gextent for a in grid_axes), *(a.glen for a in grid_axes),
            *(a.gstarts[k] for a, k in zip(grid_axes, k3)), *(t[k].data_ptr() for t, k in zip(tables, k3)),
            *(a.prev_end(k) for a, k in zip(grid_axes, k3)), *(a.next_start(k) for a, k in zip(grid_axes, k3)),
            native.stream_ptr()), "tile_blend")
        del y  # frees the tile before the next window runs
    return out


def encode(encoder: nn.Module, x: torch.Tensor, *, tile, overlap) -> torch.Tensor:
    """The blended output of `encoder` (tae.Encoder: moments [B, 2z, T/f, H/f, W/f]; ae.Encoder: [B, z, H/f, W/f]) in
    its parameters' dtype, computed over windows of `tile` samples per axis that overlap by `overlap` samples. Apply
    `reg` or the VQ quantizer afterwards. Inference only."""
    return _run(encoder, x, tile, overlap, decode=False)


def decode(decoder: nn.Module, z: torch.Tensor, *, tile, overlap) -> torch.Tensor:
    """The blended output of `decoder` ([B, out_ch, ...] at f times the latent extents) in its parameters' dtype,
    computed over latent windows of `tile` output samples per axis that overlap by `overlap` samples. Inference
    only."""
    return _run(decoder, z, tile, overlap, decode=True)
