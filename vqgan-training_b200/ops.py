"""torch.autograd.Functions over the native sm_90a kernels (libvqb200.so).

Internal activation format: contiguous bf16 tensors of shape [N, H, W, Cp] (NHWC, Cp = channels padded to a multiple
of 8, pad channels zero). Master weights / gradients stay fp32 OIHW nn.Parameters (the reference's state_dict
contract); bf16 packed copies for the tensor-core kernels are caches keyed on the parameter version. A module converted
with `.bfloat16()` (the reference's model-card inference recipe) keeps bf16 masters: it is packed from them directly,
returns bf16 at its boundary and is inference-only (its backward raises, see `inference_only`).

Every op here launches hand-written CUDA; nothing falls back to ATen for the math.
"""
from __future__ import annotations

import math
import os
import threading
import weakref
from typing import Optional

import torch

import native
import plans
from native import EPI_BIAS, EPI_MASK, EPI_RELU, EPI_RES, check, ptr, stream_ptr

_tapmap_cache = {}


def _L():
    return native.load()


def require_cuda(t: torch.Tensor):
    if not t.is_cuda:
        raise RuntimeError("vqgan-training_b200: the hot path runs on sm_90a CUDA tensors only (no CPU fallback)")


def tapmap_tensor(tapmap, device) -> torch.Tensor:
    key = (tuple(tapmap), str(device))
    t = _tapmap_cache.get(key)
    if t is None:
        t = torch.tensor(list(tapmap), dtype=torch.int32, device=device)
        _tapmap_cache[key] = t
    return t


MASTER_DTYPES = (torch.float32, torch.bfloat16)


def check_master_dtype(t: torch.Tensor, what="parameter"):
    """fp32 (training and inference) and bf16 (inference only) are the parameter dtypes the kernels read; anything else
    is refused here, before a pointer reaches a kernel that would reinterpret its memory."""
    if t.dtype not in MASTER_DTYPES:
        raise RuntimeError(f"vqgan-training_b200: {what} has dtype {t.dtype}; supported parameter dtypes are "
                           "torch.float32 (training and inference) and torch.bfloat16 (inference only)")


def inference_only(*params):
    """Backward guard of the conv / GroupNorm functions: bf16 modules are inference-only (there are no bf16-master
    gradient kernels, and the optimizer path keeps fp32 masters)."""
    for p in params:
        if p is not None and p.dtype != torch.float32:
            raise RuntimeError(
                f"vqgan-training_b200: bf16 modules are inference-only: backward through a module with {p.dtype} "
                "parameters is not supported. Run it under torch.no_grad() / torch.inference_mode(), or train the "
                "float32 module (`.float()`).")


def pack_weights(weight: torch.Tensor, tapmap, transpose: bool, Kpad: int, fold: bool = False) -> torch.Tensor:
    """OIHW fp32 or bf16 -> bf16 [R][len(tapmap)][Kpad] (R = Cin if transpose else Cout). fold: tapmap holds bit masks
    of taps whose weights are summed (fp32) before the single bf16 rounding."""
    Cout, Cin, KH, KW = weight.shape
    R = Cin if transpose else Cout
    out = torch.empty(R, len(tapmap), Kpad, device=weight.device, dtype=torch.bfloat16)
    tm = tapmap_tensor(tapmap, weight.device)
    w = weight.detach()
    if w.dtype == torch.bfloat16:
        w = w.contiguous()
        fn = _L().vqb_pack_weights_fold_bf16 if fold else _L().vqb_pack_weights_bf16
    else:
        if w.dtype != torch.float32 or not w.is_contiguous():
            w = w.float().contiguous()
        fn = _L().vqb_pack_weights_fold if fold else _L().vqb_pack_weights
    check(fn(ptr(w), ptr(out), Cout, Cin, KH * KW, len(tapmap), ptr(tm), 1 if transpose else 0, Kpad, stream_ptr()),
          "pack_weights")
    return out


class _PackEntry:
    """One cached bf16 GEMM operand of one fp32 or bf16 OIHW parameter + the recipe to rebuild it in place."""

    __slots__ = ("wref", "out", "tm", "spec", "ver", "dtype", "__weakref__")

    def __init__(self, weight, out, tm, spec):
        self.wref = weakref.ref(weight)
        self.out, self.tm, self.spec = out, tm, spec
        self.ver = (weight._version, weight.data_ptr())
        self.dtype = weight.dtype  # the master's dtype selects the kernel's source type (VqbPackJob.w_bf16)

    def job(self, first_block):
        w = self.wref()
        Cout, Cin, T, nslots, transpose, Kpad, fold, sg, ld_g, ld_r = self.spec
        return native.VqbPackJob(w=w.data_ptr(), out=self.out.data_ptr(), tapmap=self.tm.data_ptr(), Cout=Cout, Cin=Cin,
                                 T=T, nslots=nslots, transpose=transpose, Kpad=Kpad, fold=fold, sg=sg, ld_g=ld_g,
                                 ld_r=ld_r, first_block=first_block,
                                 w_bf16=1 if self.dtype == torch.bfloat16 else 0)

    def blocks(self):  # one block = an 8-row x 64-k tile, all slots (csrc/optim.cu)
        Cout, Cin, T, nslots, transpose, Kpad = self.spec[:6]
        assert T <= 16
        return -(-(Cin if transpose else Cout) // 8) * -(-Kpad // 64)

    def pack_alone(self):
        """Re-packs this entry in place with the per-tensor kernel (vqb_pack_weights[_fold][_bf16], up to 31 taps): the
        route of the 27-tap 3x3x3 weights of tae.py, which the one-launch multi-pack kernel (<= 16 taps) does not take."""
        Cout, Cin, T, nslots, transpose, Kpad, fold = self.spec[:7]
        assert self.spec[7] == nslots, "the fat-pixel layout is packed by the multi-pack kernel only"
        w = self.wref().detach()
        if self.dtype == torch.bfloat16:
            fn = _L().vqb_pack_weights_fold_bf16 if fold else _L().vqb_pack_weights_bf16
        else:
            fn = _L().vqb_pack_weights_fold if fold else _L().vqb_pack_weights
        check(fn(ptr(w), ptr(self.out), Cout, Cin, T, nslots, ptr(self.tm), transpose, Kpad, stream_ptr()),
              "pack_weights")


# taps per filter the one-launch multi-pack kernel takes (kPackMaxT in csrc/optim.cu); larger filters (the 27 taps of a
# 3x3x3 conv) are packed per tensor
PACK_MULTI_MAX_TAPS = 16


# every live pack entry, by the data_ptr of the master weight it was packed from (weak: caches own the entries)
_pack_registry = {}
_pack_tables = {}
_captured_pack_tables = []


def _new_pack_entry(weight, tapmap, transpose, Kpad, fold, fat=False) -> _PackEntry:
    Cout, Cin = weight.shape[:2]
    T = math.prod(weight.shape[2:])  # OIHW or OIDHW (tae.py's Conv3d)
    R = Cin if transpose else Cout
    nslots = len(tapmap)
    if fat:  # [R][9 slots][8] -> [R][3][64]: columns kw*8 + c of each kh row, zero beyond 24 (plans.geom_fat3)
        assert nslots == 9 and Kpad == 8
        out = torch.zeros(R, 3, plans.FAT_K, device=weight.device, dtype=torch.bfloat16)
        spec = (Cout, Cin, T, nslots, 1 if transpose else 0, Kpad, 0, 3, plans.FAT_K, 3 * plans.FAT_K)
    else:
        out = torch.empty(R, nslots, Kpad, device=weight.device, dtype=torch.bfloat16)
        spec = (Cout, Cin, T, nslots, 1 if transpose else 0, Kpad, 1 if fold else 0, nslots, 0, nslots * Kpad)
    check_master_dtype(weight, "conv master weight")
    if not weight.is_contiguous():
        raise RuntimeError("vqgan-training_b200: conv master weights must be contiguous OIHW tensors")
    ent = _PackEntry(weight, out, tapmap_tensor(tapmap, weight.device), spec)
    _pack_registry.setdefault(weight.data_ptr(), weakref.WeakSet()).add(ent)
    return ent


def _run_pack(entries):
    """Re-packs `entries` (in place) with ONE vqb_pack_weights_multi launch (fp32 and bf16 masters may be mixed: each
    job carries its source dtype); the device job table is cached per entry set. Entries of filters with more than
    PACK_MULTI_MAX_TAPS taps are packed per tensor instead."""
    alone = [e for e in entries if e.spec[2] > PACK_MULTI_MAX_TAPS]
    if alone:
        for e in alone:
            e.pack_alone()
            w = e.wref()
            e.ver = (w._version, w.data_ptr())
        entries = [e for e in entries if e.spec[2] <= PACK_MULTI_MAX_TAPS]
    if not entries:
        return
    key = tuple(id(e) for e in entries)
    tab = _pack_tables.get(key)
    if tab is None or any(r() is None for r in tab[3]):
        jobs, nb = [], 0
        for e in entries:
            jobs.append(e.job(nb))
            nb += e.blocks()
        arr = (native.VqbPackJob * len(jobs))(*jobs)
        host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
        dev = host.to(entries[0].out.device)
        if len(_pack_tables) > 64:
            _pack_tables.clear()
        tab = (dev, len(jobs), nb, [weakref.ref(e) for e in entries])
        _pack_tables[key] = tab
    if torch.cuda.is_current_stream_capturing():
        # a captured launch reads this job table on every replay: keep it alive even if the cache above is cleared
        # later (another trainer's first steps add entries), or its memory would be handed to other tensors
        _captured_pack_tables.append(tab)
    check(_L().vqb_pack_weights_multi(tab[0].data_ptr(), tab[1], tab[2], stream_ptr()), "pack_weights_multi")
    for e in entries:
        w = e.wref()
        e.ver = (w._version, w.data_ptr())


def weights_updated(params=None):
    """Call after master weights changed through a path that does not bump `Tensor._version` (fused / foreach optimizers,
    `.data` writes such as a DDP broadcast): re-packs every cached bf16 operand of `params` (all parameters if None) in
    one launch. A global optimizer post-step hook (registered below) calls this for every torch.optim optimizer."""
    if params is None:
        ptrs = list(_pack_registry.keys())
    else:
        ptrs = [p.data_ptr() for p in params]
    entries = []
    for dp in ptrs:
        ws = _pack_registry.get(dp)
        if not ws:
            continue
        for e in list(ws):
            w = e.wref()
            if w is None or w.data_ptr() != dp or w.dtype != e.dtype:
                ws.discard(e)
                continue
            entries.append(e)
        if not ws:
            _pack_registry.pop(dp, None)
    if entries:
        entries.sort(key=id)
        with torch.no_grad():
            _run_pack(entries)


def _optimizer_post_step(optimizer, args, kwargs):
    try:
        params = [p for g in optimizer.param_groups for p in g["params"] if p.is_cuda]
    except Exception:  # pragma: no cover
        params = None
    if params is None or params:
        weights_updated(params)


try:  # fused AdamW (and any .data-style update) does not bump _version: never trust the version alone (ADVICE r1, high)
    from torch.optim.optimizer import register_optimizer_step_post_hook as _reg_hook

    _reg_hook(_optimizer_post_step)
except Exception:  # pragma: no cover
    pass


class PackedCache:
    """Per-conv-layer caches: bf16 packed copies of the OIHW parameter (fp32 or bf16) and the shape-dependent geometry
    objects /
    C descriptors (built once per input shape). A packed copy is valid while (parameter version, data_ptr) are unchanged;
    updates that bypass the version counter are announced through `weights_updated` (global optimizer post-step hook)."""

    def __init__(self):
        self._store = {}
        self._geoms = {}

    def geom(self, key, builder):
        g = self._geoms.get(key)
        if g is None:
            g = builder()
            self._geoms[key] = g
        return g

    def get(self, weight: torch.Tensor, key, tapmap, transpose, Kpad, fold=False, fat=False):
        ent = self._store.get(key)
        if ent is None or ent.wref() is None or ent.ver[1] != weight.data_ptr() or ent.dtype != weight.dtype or \
                tuple(ent.out.shape[:1]) != ((weight.shape[1] if transpose else weight.shape[0]),):
            ent = _new_pack_entry(weight, tapmap, transpose, Kpad, fold, fat)
            self._store[key] = ent
            with torch.no_grad():
                _run_pack([ent])
        elif ent.ver[0] != weight._version:
            with torch.no_grad():
                _run_pack([ent])
        return ent.out


# Gradient slots: when a parameter lives in a flat.FlatParams store, the kernels that produce its gradient write straight
# into the matching slot of the store's flat gradient buffer and return that view; autograd adopts it as `param.grad`
# (no per-tensor gradient allocation, no copy-in before the all-reduce / fused optimizer).
_grad_slots = {}


def register_grad_slot(param, store, index):
    _grad_slots[param.data_ptr()] = (weakref.ref(store), index)


def grad_out(param: torch.Tensor) -> torch.Tensor:
    """fp32 destination for the gradient of `param`: its flat-store slot (first contribution of this accumulation
    window) or a fresh tensor."""
    ent = _grad_slots.get(param.data_ptr())
    if ent is not None:
        store = ent[0]()
        if store is None:
            _grad_slots.pop(param.data_ptr(), None)
        else:
            q = store.plist[ent[1]]
            if q.data_ptr() == param.data_ptr() and q.shape == param.shape:
                s = store.take_slot(ent[1])
                if s is not None:
                    return s
    return torch.empty(param.shape, device=param.device, dtype=torch.float32)


H100_SMS = 132  # H100 SXM; used when no device is visible (host-side planning and tests)


def _num_sms() -> int:
    """SM count of the current device (the kernels size their persistent grids from it), else an H100 SXM's."""
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return H100_SMS


def _wgrad_block_n(cols: int) -> int:
    """wgmma column block of csrc/wgrad_gemm.cu."""
    return 128 if cols % 128 == 0 else 64


def _wgrad_tile_blocks(cols: int) -> int:
    """Column blocks per CTA tile of csrc/wgrad_gemm.cu: two (256 columns) when the columns divide by 256."""
    return 2 if cols % 256 == 0 else 1


def choose_ksplit(g: plans.ConvGeom, Cout_pad: int) -> int:
    """Split-K factor of the weight-gradient GEMM: the split count whose (tile, split) unit count best fills whole waves
    of the persistent CTAs (one per SM of an H100 SXM), preferring one wave. Mirrors the tile shape rules of
    csrc/wgrad_gemm.cu (128 Cout rows x one or two blocks of 128 or 64 columns, 64-pixel K blocks; for a 3-D geometry, 64-voxel boxes)."""
    cols = len(g.taps) * ((g.C + 63) // 64) * 64
    rows = 128
    kpix = 64
    tiles = ((Cout_pad + rows - 1) // rows) * (cols // (_wgrad_block_n(cols) * _wgrad_tile_blocks(cols)))

    def p2(v, cap):
        p = 1
        while p < v:
            p <<= 1
        return min(p, cap)

    bw = p2(g.Wo, kpix)
    bh = p2(g.Ho, kpix // bw)
    if isinstance(g, plans.ConvGeom3d):  # vqb_wgrad3d_gemm: 64-voxel boxes [bw][bh][bt][bn]
        bt = p2(g.To, kpix // (bw * bh))
        bn = kpix // (bw * bh * bt)
        boxes = -(-g.Wo // bw) * -(-g.Ho // bh) * -(-g.To // bt) * -(-g.N // bn)
    else:
        bn = kpix // (bw * bh)
        boxes = -(-g.Wo // bw) * -(-g.Ho // bh) * -(-g.N // bn)
    # every unit pays a fixed pipeline-fill + fp32-partial-tile epilogue, and the reduction kernel reads ksplit partials:
    # each extra wave and each extra split is penalised
    sms = _num_sms()
    max_ks = max(1, min(boxes // 4, 128, (256 << 20) // max(1, Cout_pad * cols * 4)))
    best, best_score = 1, -1.0
    for ks in range(1, max_ks + 1):
        units = tiles * ks
        waves = -(-units // sms)
        eff = units / (waves * sms)
        score = eff - 0.06 * (waves - 1) - 0.0005 * ks
        if score > best_score:
            best, best_score = ks, score
    return best


def run_conv_gemm(g: plans.ConvGeom, a: torch.Tensor, wp: torch.Tensor, Cout: int, out: torch.Tensor, out_strides,
                  out_ptr_offset_bytes=0, bias=None, res=None, mask=None, relu=False, out_f32=False, stats=None):
    flags = (EPI_BIAS if bias is not None else 0) | (EPI_RES if res is not None else 0) | \
            (EPI_MASK if mask is not None else 0) | (EPI_RELU if relu else 0) | \
            (native.EPI_STATS if stats is not None else 0)
    dk = (Cout, tuple(out_strides), flags, out_f32)
    descs = g.__dict__.setdefault("_descs", {})
    d = descs.get(dk)
    if d is None:
        d = plans.conv_desc(g, Cout, out_strides, flags, out_f32)
        descs[dk] = d
    off = out_ptr_offset_bytes
    check(_L().vqb_conv_gemm(d, ptr(a), ptr(wp), ptr(bias), (ptr(res) + off) if res is not None else 0,
                             (ptr(mask) + off) if mask is not None else 0, ptr(out) + off, ptr(stats), stream_ptr()),
          "conv_gemm")


def conv_stats_supported(g: plans.ConvGeom, Cout: int, out_strides) -> bool:
    """Can the conv epilogue produce the GroupNorm statistics of its output for this geometry? (cached per geometry)"""
    descs = g.__dict__.setdefault("_descs", {})
    key = ("stats_ok", Cout, tuple(out_strides))
    ok = descs.get(key)
    if ok is None:
        ok = bool(_L().vqb_conv_stats_ok(plans.conv_desc(g, Cout, out_strides, 0, False)))
        descs[key] = ok
    return ok


def run_wgrad(g: plans.ConvGeom, x: torch.Tensor, dy: torch.Tensor, weight_shape, Cout_pad: int,
              dy_view=None, out=None) -> torch.Tensor:
    """-> OIHW fp32 gradient for a conv whose forward geometry is g (weight_shape = (Cout, K per tap, taps_h, taps_w))."""
    Cout, Cin, KH, KW = weight_shape
    wk = ("wgrad", Cout_pad, dy_view is not None)
    descs = g.__dict__.setdefault("_descs", {})
    ent = descs.get(wk)
    if ent is None:
        ksplit = choose_ksplit(g, Cout_pad)
        ent = (ksplit, plans.wgrad_desc(g, Cout_pad, ksplit, dy_view=dy_view), _L().vqb_wgrad_cols(len(g.taps), g.C))
        descs[wk] = ent
    ksplit, d, cols = ent
    partial = torch.empty(ksplit, Cout_pad, cols, device=x.device, dtype=torch.float32)
    check(_L().vqb_wgrad_gemm(d, ptr(dy), ptr(x), ptr(partial), stream_ptr()), "wgrad_gemm")
    grad = out if out is not None else torch.empty(Cout, Cin, KH, KW, device=x.device, dtype=torch.float32)
    assert grad.shape == (Cout, Cin, KH, KW) and grad.is_contiguous()
    tm = tapmap_tensor(g.tapmap if len(g.tapmap) == len(g.taps) else list(range(len(g.taps))), x.device)
    check(_L().vqb_wgrad_reduce(ptr(partial), ptr(grad), ksplit, Cout, Cout_pad, Cin, KH * KW, len(g.taps),
                                cols // len(g.taps), ptr(tm), 0, stream_ptr()), "wgrad_reduce")
    return grad


# One-slot side channel from GroupNormSiLUFn.backward to the backward of the conv that produced the normalised tensor:
# the GN backward apply pass already streams dx (= that conv's dy), so it also emits the per-channel sums (= the conv's
# bias gradient). The slot holds a strong reference to dx, so a matching data_ptr can only be that very tensor; the
# version check rejects a tensor that autograd accumulated into in place. Any mismatch falls back to vqb_colsum.
class _Slot(threading.local):
    """one slot per thread: autograd runs a device's backward on one worker thread, so a re-entrant or concurrent
    backward on another thread can neither see nor clobber this one's hand-over"""

    def __init__(self):
        self.v = None

    def __getitem__(self, i):
        return self.v

    def __setitem__(self, i, val):
        self.v = val


_dx_colsum_slot = _Slot()


def _take_dx_colsum(dy: torch.Tensor, C: int):
    ent = _dx_colsum_slot[0]
    if ent is None:
        return None
    t, ver, cs = ent
    if (t.data_ptr() == dy.data_ptr() and t.shape == dy.shape and t.stride() == dy.stride() and t.dtype == dy.dtype
            and dy._version == ver and cs.numel() == C):
        _dx_colsum_slot[0] = None
        return cs
    return None


def colsum(x2d_rows: int, x: torch.Tensor, C: int, out=None) -> torch.Tensor:
    if out is None:
        out = torch.empty(C, device=x.device, dtype=torch.float32)
    check(_L().vqb_colsum(ptr(x), ptr(out), x2d_rows, C, stream_ptr()), "colsum")
    return out


# ----------------------------------------------------------------------------------------------------------------------
class ToNHWC(torch.autograd.Function):
    """[N,C,H,W] fp32 or bf16 -> [N,H,W,Cp] bf16, optional per-channel (x - shift) * inv_scale (LPIPS ScalingLayer,
    utils.py:70-71). A bf16 input is read directly (no fp32 copy). Backward: NHWC bf16 grad -> NCHW fp32 (* inv_scale)."""

    @staticmethod
    def forward(ctx, x, shift, inv_scale, frame):
        require_cuda(x)
        x = x.detach()
        bf16 = x.dtype == torch.bfloat16
        if bf16:
            x = x.contiguous()
        elif x.dtype != torch.float32 or not x.is_contiguous():
            x = x.float().contiguous()
        N, C, H, W = x.shape
        Cp = plans.cpad(C)
        if frame:  # zero-framed [N, H+2, W+2, Cp] for the "fat pixel" first-layer conv
            y = alloc_framed(N, H, W, Cp, x.device)
            fn = _L().vqb_nchw_to_nhwc_pad_bf16 if bf16 else _L().vqb_nchw_to_nhwc_pad
            check(fn(ptr(x), ptr(y), N, C, H, W, Cp, 1, ptr(shift), ptr(inv_scale), stream_ptr()), "nchw_to_nhwc_pad")
        else:
            y = torch.empty(N, H, W, Cp, device=x.device, dtype=torch.bfloat16)
            fn = _L().vqb_nchw_to_nhwc_bf16 if bf16 else _L().vqb_nchw_to_nhwc
            check(fn(ptr(x), ptr(y), N, C, H, W, Cp, ptr(shift), ptr(inv_scale), stream_ptr()), "nchw_to_nhwc")
        ctx.shape = (N, C, H, W, Cp)
        ctx.inv_scale, ctx.frame = inv_scale, frame
        return y

    @staticmethod
    def backward(ctx, gy):
        N, C, H, W, Cp = ctx.shape
        gy = gy.contiguous()
        gx = torch.empty(N, C, H, W, device=gy.device, dtype=torch.float32)
        if ctx.frame:
            check(_L().vqb_nhwc_to_nchw_pad(ptr(gy), ptr(gx), N, C, H, W, Cp, 1, ptr(ctx.inv_scale), stream_ptr()),
                  "nhwc_to_nchw_pad")
        else:
            check(_L().vqb_nhwc_to_nchw(ptr(gy), ptr(gx), N, C, H, W, Cp, ptr(ctx.inv_scale), stream_ptr()),
                  "nhwc_to_nchw")
        return gx, None, None, None


def alloc_framed(N, H, W, C, device) -> torch.Tensor:
    """Zeroed [N, H+2, W+2, C] bf16 buffer followed by 64 elements of zeroed slack (fat-pixel K runs read up to 5 pixels
    past the last one; they meet zero weights but must stay inside the allocation and finite)."""
    n = N * (H + 2) * (W + 2) * C
    return torch.zeros(n + 64, device=device, dtype=torch.bfloat16)[:n].view(N, H + 2, W + 2, C)


def _fat_weights(cache: "PackedCache", weight, key, tapmap, transpose, Kpad):
    """[R][9 slots][8] packing laid out as [R][3][64]: columns kw*8 + c of each kh row, zero beyond 24 (plans.geom_fat3)."""
    return cache.get(weight, tuple(key) + ("k64",), tapmap, transpose, Kpad, fat=True)


_fat_state = {"ok": None}


def fat_conv_enabled() -> bool:
    """One-time self check of the fat-pixel first-layer path (it relies on a TMA map whose pixel stride (16 B) is smaller
    than its 48-byte inner extent): run a tiny conv both ways; disable the path on any error or mismatch."""
    if _fat_state["ok"] is None:
        _fat_state["ok"] = False
        # normal tensors even when the first caller runs under torch.inference_mode() (the pack cache reads _version)
        try:
            with torch.inference_mode(False):
                g = torch.Generator(device="cuda").manual_seed(1)
                x = torch.rand(2, 3, 16, 24, device="cuda", generator=g) - 0.5
                w = torch.rand(64, 3, 3, 3, device="cuda", generator=g) - 0.5
                c1, c2 = PackedCache(), PackedCache()
                a = conv(ToNHWC.apply(x, None, None, False), w, None, c1, "s1")
                b = conv(ToNHWC.apply(x, None, None, True), w, None, c2, "fat3")
                torch.cuda.synchronize()
                _fat_state["ok"] = bool(torch.allclose(a.float(), b.float(), rtol=2e-2, atol=2e-2))
        except Exception:
            _fat_state["ok"] = False
    return _fat_state["ok"]


def wavelet_to_nhwc(x: torch.Tensor, filt: torch.Tensor) -> torch.Tensor:
    """[N,C,H,W] fp32 or bf16 image -> [N,H/2,W/2,cpad(4C)] bf16: the wavelet front-end (utils.py:229-247) fused with the
    layout conversion. Input-side op: the image is data, so there is no backward."""
    require_cuda(x)
    if x.requires_grad:
        raise RuntimeError("wavelet front-end: the input image must not require grad (input-side op without backward)")
    bf16 = x.dtype == torch.bfloat16
    x = x.detach().contiguous() if bf16 else x.detach().float().contiguous()
    N, C, H, W = x.shape
    Cp = plans.cpad(4 * C)
    y = torch.empty(N, H // 2, W // 2, Cp, device=x.device, dtype=torch.bfloat16)
    f = filt.detach().to(device=x.device, dtype=torch.float32).reshape(4, 36).contiguous()
    fn = _L().vqb_wavelet_fwd_bf16 if bf16 else _L().vqb_wavelet_fwd
    check(fn(ptr(x), ptr(y), ptr(f), N, C, H, W, Cp, stream_ptr()), "wavelet_fwd")
    return y


def to_nhwc(x, shift=None, inv_scale=None, frame=False):
    return ToNHWC.apply(x, shift, inv_scale, frame)


def clip_frame_selection(frames, B: int, T: int):
    """Host-side check of a frame selection for [B, C, T, H, W] clips: None (every frame) or a [B, T'] integer tensor or
    nested list holding T' distinct frames in [0, T) per clip. -> (int32 CPU tensor [B*T'] or None, T'). Raises before
    anything is launched; a CUDA tensor is copied to the host (one synchronisation)."""
    if frames is None:
        return None, T
    f = torch.as_tensor(frames)
    if f.is_floating_point() or f.is_complex() or f.dtype == torch.bool:
        raise ValueError(f"frames must be integers, got {f.dtype}")
    if f.dim() != 2 or f.shape[0] != B or not 1 <= f.shape[1] <= T:
        raise ValueError(f"frames must be a [B, T'] selection with B = {B} and 1 <= T' <= T = {T}, got shape "
                         f"{tuple(f.shape)}")
    f = f.to("cpu", torch.int64)
    if bool(((f < 0) | (f >= T)).any()):
        raise ValueError(f"frames holds a frame outside [0, {T}): {f.tolist()}")
    if bool((f.sort(dim=1).values.diff(dim=1) == 0).any()):
        raise ValueError(f"frames holds a duplicate frame within a clip: {f.tolist()}")
    return f.to(torch.int32).reshape(-1), f.shape[1]


class ClipToFrames(torch.autograd.Function):
    """The clip counterpart of ToNHWC: [B,C,T,H,W] fp32 or bf16 -> [B*T', H, W, Cp] bf16 (zero-framed [B*T', H+2, W+2,
    Cp] with frame=True), frames folded into the batch in (b, t) order, optional (x - shift) * inv_scale. `sel` is the
    int32 CPU [B*T'] selection of clip_frame_selection (None: every frame). The clip is read through its strides, with
    no folded copy; each image is bit-identical to ToNHWC of that frame. Backward: the NCTHW fp32 clip gradient
    (* inv_scale), exact zeros in frames outside the selection, from one launch."""

    @staticmethod
    def forward(ctx, x, shift, inv_scale, frame, sel, Tsel):
        require_cuda(x)
        x = x.detach()
        bf16 = x.dtype == torch.bfloat16
        if bf16:
            x = x.contiguous()
        elif x.dtype != torch.float32 or not x.is_contiguous():
            x = x.float().contiguous()
        B, C, T, H, W = x.shape
        Cp = plans.cpad(C)
        # pinned + non_blocking: a pageable host-to-device copy would wait for the stream to drain
        sel_dev = None if sel is None else sel.pin_memory().to(x.device, non_blocking=True)
        if frame:
            y = alloc_framed(B * Tsel, H, W, Cp, x.device)
            fn = _L().vqb_ncthw_frames_to_nhwc_pad_bf16 if bf16 else _L().vqb_ncthw_frames_to_nhwc_pad
            check(fn(ptr(x), ptr(y), B, C, T, H, W, Cp, 1, ptr(sel_dev), Tsel, ptr(shift), ptr(inv_scale),
                     stream_ptr()), "ncthw_frames_to_nhwc_pad")
        else:
            y = torch.empty(B * Tsel, H, W, Cp, device=x.device, dtype=torch.bfloat16)
            fn = _L().vqb_ncthw_frames_to_nhwc_bf16 if bf16 else _L().vqb_ncthw_frames_to_nhwc
            check(fn(ptr(x), ptr(y), B, C, T, H, W, Cp, ptr(sel_dev), Tsel, ptr(shift), ptr(inv_scale), stream_ptr()),
                  "ncthw_frames_to_nhwc")
        ctx.shape = (B, C, T, H, W, Cp, Tsel)
        ctx.inv_scale, ctx.frame, ctx.sel_dev = inv_scale, frame, sel_dev
        return y

    @staticmethod
    def backward(ctx, gy):
        B, C, T, H, W, Cp, Tsel = ctx.shape
        gy = gy.contiguous()
        gx = torch.empty(B, C, T, H, W, device=gy.device, dtype=torch.float32)
        if ctx.frame:
            check(_L().vqb_nhwc_pad_frames_to_ncthw(ptr(gy), ptr(gx), B, C, T, H, W, Cp, 1, ptr(ctx.sel_dev), Tsel,
                                                    ptr(ctx.inv_scale), stream_ptr()), "nhwc_pad_frames_to_ncthw")
        else:
            check(_L().vqb_nhwc_frames_to_ncthw(ptr(gy), ptr(gx), B, C, T, H, W, Cp, ptr(ctx.sel_dev), Tsel,
                                                ptr(ctx.inv_scale), stream_ptr()), "nhwc_frames_to_ncthw")
        return gx, None, None, None, None, None


def clip_to_frames(x, shift=None, inv_scale=None, frame=False, frames=None):
    """[B,C,T,H,W] clip -> per-frame NHWC bf16 images of the selected frames (ClipToFrames; frames as in
    clip_frame_selection)."""
    if x.dim() != 5:
        raise ValueError(f"clip_to_frames: expected a [B, C, T, H, W] clip, got shape {tuple(x.shape)}")
    sel, Tsel = clip_frame_selection(frames, x.shape[0], x.shape[2])
    return ClipToFrames.apply(x, shift, inv_scale, frame, sel, Tsel)


class ToNCHW(torch.autograd.Function):
    """[N,H,W,Cp] bf16 -> [N,C,H,W] fp32, or bf16 for a bf16 module (module-boundary output when a caller wants the
    reference layout)."""

    @staticmethod
    def forward(ctx, y, C, dtype=torch.float32):
        N, H, W, Cp = y.shape
        y = y.contiguous()
        if dtype == torch.bfloat16:
            x = torch.empty(N, C, H, W, device=y.device, dtype=torch.bfloat16)
            check(_L().vqb_nhwc_to_nchw_bf16(ptr(y), ptr(x), N, C, H, W, Cp, stream_ptr()), "nhwc_to_nchw_bf16")
        else:
            x = torch.empty(N, C, H, W, device=y.device, dtype=torch.float32)
            check(_L().vqb_nhwc_to_nchw(ptr(y), ptr(x), N, C, H, W, Cp, 0, stream_ptr()), "nhwc_to_nchw")
        ctx.shape = (N, C, H, W, Cp)
        return x

    @staticmethod
    def backward(ctx, gx):
        N, C, H, W, Cp = ctx.shape
        gx = gx.float().contiguous()
        gy = torch.empty(N, H, W, Cp, device=gx.device, dtype=torch.bfloat16)
        check(_L().vqb_nchw_to_nhwc(ptr(gx), ptr(gy), N, C, H, W, Cp, 0, 0, stream_ptr()), "nchw_to_nhwc")
        return gy, None, None


def to_nchw(y, C, dtype=torch.float32):
    """dtype: the dtype of the module's parameters (fp32 or bf16), which is what the reference returns."""
    return ToNCHW.apply(y, C, dtype)


# ----------------------------------------------------------------------------------------------------------------------
class ConvFn(torch.autograd.Function):
    """Convolution through the wgmma implicit-GEMM kernel.

    kind: "s1" (k x k stride 1 same), "s2" (Downsample: pad (0,1,0,1) + 3x3 stride 2), "patch" (k x k stride k).
    opts: relu (fused ReLU epilogue; the incoming gradient is then expected to be already gated by out > 0, which every
    consumer of a ReLU output in this package does), input_is_relu (gate the data gradient by x > 0 in the dgrad
    epilogue), nchw_out (write [N,Cout,H,W] in the weight's dtype, fp32 or bf16, directly: encoder z / decoder image)."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, cache, kind, relu, input_is_relu, nchw_out, want_stats=False):
        require_cuda(x)
        N, H, W, Cp = x.shape
        Cout, Cin, KH, KW = weight.shape
        assert Cp == plans.cpad(Cin), f"conv input has {Cp} channels, weight expects {Cin}"
        x = x.contiguous()
        if kind == "fat3":
            assert Cp == 8 and KH == 3
        g, H, W = _conv_geom(cache, kind, N, H, W, Cp, KH)
        if kind == "fat3":
            wp = _fat_weights(cache, weight, ("fwd", kind), g.tapmap, False, Cp)
        else:
            wp = cache.get(weight, ("fwd", kind), g.tapmap, False, Cp)
        Cop = plans.cpad(Cout)
        b = None
        if bias is not None:
            b = bias.detach()
            if b.dtype != torch.float32:
                b = b.float()
        if nchw_out:  # a bf16 module's z / image: the epilogue's strided bf16 store (out_f32 = 0, oc = H*W)
            f32 = weight.dtype == torch.float32
            out = torch.empty(N, Cout, g.Ho, g.Wo, device=x.device, dtype=torch.float32 if f32 else torch.bfloat16)
            run_conv_gemm(g, x, wp, Cout, out, plans.nchw_strides(Cout, g.Ho, g.Wo), bias=b, relu=relu, out_f32=f32)
        else:
            alloc = torch.empty if Cop == Cout else torch.zeros
            out = alloc(N, g.Ho, g.Wo, Cop, device=x.device, dtype=torch.bfloat16)
            res = residual.contiguous() if residual is not None else None
            ostr = plans.nhwc_strides(g.Ho, g.Wo, Cop)
            stats = None
            if want_stats and Cop == Cout and conv_stats_supported(g, Cout, ostr):
                stats = torch.zeros(N, Cout, 2, device=x.device, dtype=torch.float32)
            run_conv_gemm(g, x, wp, Cout, out, ostr, bias=b, res=res, relu=relu, stats=stats)
        ctx.save_for_backward(x, weight)
        ctx.cache, ctx.kind = cache, kind
        ctx.has_bias, ctx.has_res = bias is not None, residual is not None
        ctx.input_is_relu, ctx.nchw_out = input_is_relu, nchw_out
        if want_stats and not nchw_out:
            if stats is None:
                stats = torch.empty(0, device=x.device)  # "not available" marker
            ctx.mark_non_differentiable(stats)
            return out, stats
        return out

    @staticmethod
    def backward(ctx, gout, _gstats=None):
        x, weight = ctx.saved_tensors
        inference_only(weight)
        gx, gw, gb, gres = conv_backward(x, weight, gout, ctx.cache, ctx.kind, ctx.has_bias, ctx.has_res,
                                         ctx.input_is_relu, ctx.nchw_out, ctx.needs_input_grad[:4])
        return gx, gw, gb, gres, None, None, None, None, None, None


def _conv_geom(cache, kind, N, H, W, Cp, KH):
    """-> (forward geometry, H, W) of conv kind `kind` over an [N, H, W, Cp] input; for "fat3" the input is the
    zero-framed [N, H+2, W+2, 8] image and H, W are those of the image inside the frame."""
    if kind == "fat3":
        H, W = H - 2, W - 2
        return cache.geom(("fat", N, H, W), lambda: plans.geom_fat3(N, H, W)), H, W
    if kind == "s1":
        return cache.geom(("f", N, H, W), lambda: plans.geom_s1(N, H, W, Cp, KH)), H, W
    if kind == "s2":
        return cache.geom(("f", N, H, W), lambda: plans.geom_s2(N, H, W, Cp)), H, W
    if kind == "patch":
        return cache.geom(("f", N, H, W), lambda: plans.geom_patch(N, H, W, Cp, KH)), H, W
    raise ValueError(kind)


def conv_backward(x, weight, gout, cache, kind, has_bias, has_res, input_is_relu, nchw_out, needs):
    """Backward of conv(x, weight, bias, cache, kind, residual, relu, input_is_relu, nchw_out) from its input x, its
    weight and the incoming gradient -> (gx, gw, gb, gres); needs: which of (x, weight, bias, residual) want a
    gradient."""
    N, H, W, Cp = x.shape
    Cout, Cin, KH, KW = weight.shape
    g, H, W = _conv_geom(cache, kind, N, H, W, Cp, KH)
    Cop = plans.cpad(Cout)
    dy_framed = False
    if nchw_out:
        gn = gout.float().contiguous()
        if Cop == 8 and KH == 3 and kind == "s1" and fat_conv_enabled():
            # tiny-Cout conv (decoder conv_out): keep dy in a zero-framed buffer so that the data gradient runs as a
            # 3-tap fat-pixel conv (24-wide K runs) instead of 9 taps of 8 channels
            dy_framed = True
            dy = alloc_framed(N, g.Ho, g.Wo, Cop, x.device)
            check(_L().vqb_nchw_to_nhwc_pad(ptr(gn), ptr(dy), N, Cout, g.Ho, g.Wo, Cop, 1, 0, 0, stream_ptr()),
                  "nchw_to_nhwc_pad")
        else:
            dy = torch.empty(N, g.Ho, g.Wo, Cop, device=x.device, dtype=torch.bfloat16)
            check(_L().vqb_nchw_to_nhwc(ptr(gn), ptr(dy), N, Cout, g.Ho, g.Wo, Cop, 0, 0, stream_ptr()),
                  "nchw_to_nhwc")
    else:
        dy = gout.contiguous()
    gx = gw = gb = gres = None
    if needs[0]:
        mask = x if input_is_relu else None
        gx_alloc = torch.empty if Cp == Cin else torch.zeros
        if kind == "fat3":  # gradient w.r.t. the framed image: write the interior of a zero-framed buffer
            gx = torch.zeros(N, H + 2, W + 2, Cp, device=x.device, dtype=torch.bfloat16)
            gd = cache.geom(("d", N, H, W), lambda: plans.geom_s1_dgrad(N, H, W, Cop, KH))
            wpd = cache.get(weight, ("dgrad", "s1"), gd.tapmap, True, Cop)
            run_conv_gemm(gd, dy, wpd, Cin, gx, ((H + 2) * (W + 2) * Cp, (W + 2) * Cp, Cp, 1),
                          out_ptr_offset_bytes=((W + 2) + 1) * Cp * 2)
        elif dy_framed:
            gx = gx_alloc(N, H, W, Cp, device=x.device, dtype=torch.bfloat16)
            gdf = cache.geom(("dfat", N, H, W), lambda: plans.geom_fat3(N, H, W, dgrad=True))
            wpd = _fat_weights(cache, weight, ("dgrad", "fat3"), gdf.tapmap, True, Cop)
            run_conv_gemm(gdf, dy, wpd, Cin, gx, plans.nhwc_strides(H, W, Cp), mask=mask)
        else:
            gx = gx_alloc(N, H, W, Cp, device=x.device, dtype=torch.bfloat16)
        if kind == "fat3" or dy_framed:
            pass
        elif kind == "s1":
            gd = cache.geom(("d", N, H, W), lambda: plans.geom_s1_dgrad(N, H, W, Cop, KH))
            wpd = cache.get(weight, ("dgrad", kind), gd.tapmap, True, Cop)
            run_conv_gemm(gd, dy, wpd, Cin, gx, plans.nhwc_strides(H, W, Cp), mask=mask)
        elif kind == "s2":
            for ph, pw, gd in cache.geom(("d", N, H, W), lambda: plans.geom_s2_dgrad_classes(N, H, W, Cop)):
                wpd = cache.get(weight, ("dgrad", kind, ph, pw), gd.tapmap, True, Cop)
                run_conv_gemm(gd, dy, wpd, Cin, gx, (H * W * Cp, 2 * W * Cp, 2 * Cp, 1),
                              out_ptr_offset_bytes=(ph * W + pw) * Cp * 2, mask=mask)
        elif kind == "patch":
            # non-overlapping windows: each input pixel belongs to exactly one (output pixel, tap): one 1-tap
            # "conv" per tap writing the strided sub-grid of dx
            k = KH
            for kh in range(k):
                for kw in range(k):
                    gd = cache.geom(("d", N, H, W, kh, kw), lambda: plans.ConvGeom(
                        N, g.Ho, g.Wo, Cop, [native.dense_view(N, g.Ho, g.Wo, Cop)], [(0, 0, 0)], [kh * k + kw]))
                    wpd = cache.get(weight, ("dgrad", kind, kh, kw), gd.tapmap, True, Cop)
                    run_conv_gemm(gd, dy, wpd, Cin, gx, (H * W * Cp, k * W * Cp, k * Cp, 1),
                                  out_ptr_offset_bytes=(kh * W + kw) * Cp * 2, mask=mask)
    if needs[1]:
        if kind == "fat3":  # [Cout][kw*8 + c][kh] -> OIHW
            g3 = run_wgrad(g, x, dy, (Cout, plans.FAT_K, 3, 1), Cop)  # [Cout][kw*8 + c (24 real of 64)][kh]
            gw = g3[:, :24, :, 0].reshape(Cout, 3, 8, 3)[:, :, :Cin, :].permute(0, 2, 3, 1).contiguous()
        elif dy_framed:
            gw = run_wgrad(g, x, dy, weight.shape, Cop,
                           dy_view=plans.framed_interior_view(N, g.Ho, g.Wo, Cop), out=grad_out(weight))
        else:
            gw = run_wgrad(g, x, dy, weight.shape, Cop, out=grad_out(weight))
    if has_bias and needs[2]:
        rows = N * (g.Ho + 2) * (g.Wo + 2) if dy_framed else N * g.Ho * g.Wo  # the zero frame adds nothing
        gb = None if dy_framed else _take_dx_colsum(dy, Cop)
        if gb is None:
            gb = colsum(rows, dy, Cop)[:Cout]
    if has_res and needs[3]:
        gres = dy
    return gx, gw, gb, gres


def conv(x, weight, bias, cache, kind="s1", residual=None, relu=False, input_is_relu=False, nchw_out=False,
         want_stats=False):
    """-> out, or (out, stats) when want_stats (stats is None if the epilogue cannot produce them for this shape)."""
    if want_stats and not nchw_out:
        out, st = ConvFn.apply(x, weight, bias, residual, cache, kind, relu, input_is_relu, nchw_out, True)
        return out, (st if st.numel() > 0 else None)
    return ConvFn.apply(x, weight, bias, residual, cache, kind, relu, input_is_relu, nchw_out, False)


# ----------------------------------------------------------------------------------------------------------------------
class UpConvFn(torch.autograd.Function):
    """Upsample (nearest x2, ae.py:165) + conv3x3 p1 (ae.py:166) without materialising the 4x tensor: four phase convs with
    2x2 folded taps over the low-res input (4/9 of the MACs; SURVEY.md Appendix A). Backward: one 16-tap conv over the
    four parity views of dy (data gradient) and four phase weight-gradient GEMMs unfolded by vqb_wgrad_reduce_fold."""

    @staticmethod
    def forward(ctx, x, weight, bias, cache, want_stats=False):
        require_cuda(x)
        x = x.contiguous()
        N, h, w, Cp = x.shape
        Cout, Cin, KH, KW = weight.shape
        assert KH == 3 and KW == 3 and Cp == plans.cpad(Cin)
        Cop = plans.cpad(Cout)
        alloc = torch.empty if Cop == Cout else torch.zeros
        out = alloc(N, 2 * h, 2 * w, Cop, device=x.device, dtype=torch.bfloat16)
        b = bias.detach().float() if bias is not None else None
        strides = (4 * h * w * Cop, 2 * 2 * w * Cop, 2 * Cop, 1)
        stats = None
        g00 = cache.geom(("uf", N, h, w, 0, 0), lambda: plans.geom_up_fwd(N, h, w, Cp, 0, 0))
        if want_stats and Cop == Cout and conv_stats_supported(g00, Cout, strides):
            stats = torch.zeros(N, Cout, 2, device=x.device, dtype=torch.float32)  # the 4 phase launches accumulate
        for ph in range(2):
            for pw in range(2):
                g = cache.geom(("uf", N, h, w, ph, pw), lambda: plans.geom_up_fwd(N, h, w, Cp, ph, pw))
                wp = cache.get(weight, ("ufwd", ph, pw), g.tapmask, False, Cp, fold=True)
                run_conv_gemm(g, x, wp, Cout, out, strides, out_ptr_offset_bytes=(ph * 2 * w + pw) * Cop * 2, bias=b,
                              stats=stats)
        ctx.save_for_backward(x, weight)
        ctx.cache, ctx.has_bias = cache, bias is not None
        if want_stats:
            if stats is None:
                stats = torch.empty(0, device=x.device)
            ctx.mark_non_differentiable(stats)
            return out, stats
        return out

    @staticmethod
    def backward(ctx, gout, _gstats=None):
        x, weight = ctx.saved_tensors
        inference_only(weight)
        cache = ctx.cache
        N, h, w, Cp = x.shape
        Cout, Cin, KH, KW = weight.shape
        Cop = plans.cpad(Cout)
        dy = gout.contiguous()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gd = cache.geom(("ud", N, h, w), lambda: plans.geom_up_dgrad(N, h, w, Cop))
            wpd = cache.get(weight, ("udgrad",), gd.tapmask, True, Cop, fold=True)
            gx_alloc = torch.empty if Cp == Cin else torch.zeros
            gx = gx_alloc(N, h, w, Cp, device=x.device, dtype=torch.bfloat16)
            run_conv_gemm(gd, dy, wpd, Cin, gx, plans.nhwc_strides(h, w, Cp))
        if ctx.needs_input_grad[1]:
            C64 = ((Cp + 63) // 64) * 64
            g00 = cache.geom(("uf", N, h, w, 0, 0), lambda: plans.geom_up_fwd(N, h, w, Cp, 0, 0))
            ksplit = choose_ksplit(g00, Cop)
            partial = torch.empty(ksplit, Cop, 16 * C64, device=x.device, dtype=torch.float32)
            masks = []
            for ph in range(2):
                for pw in range(2):
                    g = cache.geom(("uf", N, h, w, ph, pw), lambda: plans.geom_up_fwd(N, h, w, Cp, ph, pw))
                    dk = ("uwgrad", Cop, ksplit)
                    descs = g.__dict__.setdefault("_descs", {})
                    d = descs.get(dk)
                    if d is None:
                        d = plans.wgrad_desc(g, Cop, ksplit, dy_view=plans.up_dy_view(N, h, w, Cop, ph, pw),
                                             ld_override=16 * C64, col_offset=(ph * 2 + pw) * 4 * C64)
                        descs[dk] = d
                    check(_L().vqb_wgrad_gemm(d, ptr(dy), ptr(x), ptr(partial), stream_ptr()), "wgrad_gemm(up)")
                    masks += g.tapmask
            gw = grad_out(weight)
            tm = tapmap_tensor(masks, x.device)
            check(_L().vqb_wgrad_reduce_fold(ptr(partial), ptr(gw), ksplit, Cout, Cop, Cin, 9, 16, C64, ptr(tm),
                                             stream_ptr()), "wgrad_reduce_fold")
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = _take_dx_colsum(dy, Cop)
            if gb is None:
                gb = colsum(N * 4 * h * w, dy, Cop)[:Cout]
        return gx, gw, gb, None, None


def upsample_conv(x, weight, bias, cache, want_stats=False):
    if want_stats:
        out, st = UpConvFn.apply(x, weight, bias, cache, True)
        return out, (st if st.numel() > 0 else None)
    return UpConvFn.apply(x, weight, bias, cache, False)


# activation codes of the GroupNorm kernels (the `silu` argument of vqb_gn_silu_*): a bool passes as 0 / 1
ACT_NONE, ACT_SWISH, ACT_LEAKY = 0, 1, 2


class GroupNormSiLUFn(torch.autograd.Function):
    """FP32GroupNorm (32 groups, eps 1e-6, biased variance, fp32 statistics; ae.py:41-53) fused with swish
    (ae.py:13-14): one statistics pass + one apply pass over bf16 NHWC, instead of cast/GN/cast/sigmoid/mul.
    `silu` is an activation code (ACT_NONE, ACT_SWISH, ACT_LEAKY = LeakyReLU(0.2)); False / True are codes 0 / 1.

    with_skip=True additionally returns the input itself as a second output (the ResnetBlock skip connection): the
    gradient arriving through that output is summed into dx INSIDE the backward apply kernel instead of by a separate
    autograd accumulation kernel."""

    @staticmethod
    def forward(ctx, x, gamma, beta, groups, eps, silu, with_skip, chsums=None):
        require_cuda(x)
        x = x.contiguous()
        if chsums is not None:  # statistics were accumulated by the epilogue of the conv that produced x
            y, mr = gn_silu_fwd_pre(x, gamma, beta, chsums, groups, eps, silu)
        else:
            y, mr = gn_silu_fwd(x, gamma, beta, groups, eps, silu)
        ctx.save_for_backward(x, gamma, beta, mr)
        ctx.groups, ctx.silu, ctx.with_skip = groups, silu, with_skip
        ctx.set_materialize_grads(False)  # an unused output arrives as None, not as a zero tensor
        if with_skip:
            return y, x.view_as(x)
        return y

    @staticmethod
    def backward(ctx, gy, gskip=None):
        x, gamma, beta, mr = ctx.saved_tensors
        inference_only(gamma, beta)
        if gy is None:  # only the skip output was used
            return (gskip, None, None, None, None, None, None, None)
        dx, dg, db = gn_silu_bwd(x, gy, gskip, gamma, beta, mr, ctx.groups, ctx.silu)
        return dx, dg, db, None, None, None, None, None


def gn_silu_fwd(x, gamma, beta, groups, eps, silu):
    """GroupNorm(+swish) of a contiguous bf16 NHWC x through the deterministic statistics pass -> (y, mr), where
    mr [N, groups, 2] holds the (mean, rstd) the backward and gn_silu_apply take."""
    N, H, W, C = x.shape
    y = torch.empty_like(x)
    mr = torch.empty(N, groups, 2, device=x.device, dtype=torch.float32)
    ga, be = gamma.detach().float(), beta.detach().float()
    ws = torch.empty(N * C * 2, device=x.device, dtype=torch.float64)
    check(_L().vqb_gn_silu_fwd(ptr(x), ptr(y), ptr(ga), ptr(be), ptr(mr), ptr(ws), N, H * W, C, groups, eps,
                               int(silu), stream_ptr()), "gn_silu_fwd")
    return y, mr


def gn_silu_fwd_pre(x, gamma, beta, chsums, groups, eps, silu):
    """GroupNorm(+swish) of a contiguous bf16 NHWC x from the per-(n, channel) sums [N, C, 2] that the epilogue of the
    conv producing x accumulated (VQB_EPI_STATS) -> (y, mr), as gn_silu_fwd."""
    N, H, W, C = x.shape
    y = torch.empty_like(x)
    mr = torch.empty(N, groups, 2, device=x.device, dtype=torch.float32)
    ga, be = gamma.detach().float(), beta.detach().float()
    check(_L().vqb_gn_silu_fwd_pre(ptr(x), ptr(y), ptr(ga), ptr(be), ptr(mr), ptr(chsums), N, H * W, C, groups, eps,
                                   int(silu), stream_ptr()), "gn_silu_fwd_pre")
    return y, mr


def gn_silu_apply(x, gamma, beta, mr, silu):
    """The apply pass of gn_silu_fwd or gn_silu_fwd_pre alone, with that call's mr: the same y, bit for bit
    (vqb_gn_silu_apply)."""
    N, H, W, C = x.shape
    y = torch.empty_like(x)
    ga, be = gamma.detach().float(), beta.detach().float()
    check(_L().vqb_gn_silu_apply(ptr(x), ptr(y), ptr(ga), ptr(be), ptr(mr), N, H * W, C, mr.shape[1],
                                 1 if silu else 0, stream_ptr()), "gn_silu_apply")
    return y


def gn_silu_bwd(x, gy, gskip, gamma, beta, mr, groups, silu):
    """GroupNorm(+swish) backward -> (dx, dgamma, dbeta); gskip (optional) is summed into dx. The per-channel sums of dx
    are left in the colsum slot for the bias gradient of the conv that produced x."""
    N, H, W, C = x.shape
    gy = gy.contiguous()
    add = gskip.contiguous() if gskip is not None else None
    dx = torch.empty_like(x)
    dg, db = grad_out(gamma), grad_out(beta)
    ws = torch.empty(N * C * 2 + N * groups * 2, device=x.device, dtype=torch.float32)
    ga, be = gamma.detach().float(), beta.detach().float()
    cs = torch.empty(C, device=x.device, dtype=torch.float32)
    check(_L().vqb_gn_silu_bwd(ptr(x), ptr(gy), ptr(add), ptr(dx), ptr(ga), ptr(be), ptr(mr), ptr(dg), ptr(db),
                               ptr(ws), N, H * W, C, groups, int(silu), ptr(cs), stream_ptr()), "gn_silu_bwd")
    _dx_colsum_slot[0] = (dx, dx._version, cs)
    return dx, dg, db


def group_norm_silu(x, gamma, beta, groups=32, eps=1e-6, silu=True, with_skip=False, chsums=None):
    return GroupNormSiLUFn.apply(x, gamma, beta, groups, eps, silu, with_skip, chsums)


class ResnetBlockRecomputeFn(torch.autograd.Function):
    """ae.ResnetBlock as one autograd node that keeps only its input x, the two GroupNorm (mean, rstd) records and its
    parameters for the backward, instead of x, hn = swish(norm1(x)), h = conv1(hn) and h2 = swish(norm2(h)).

    The forward runs the kernels of the block's non-recomputing training forward: norm1 from the column sums chsums of
    the conv that produced x when it accumulated them (else the statistics pass), conv1 with the statistics epilogue
    where the shape allows it and norm2 from its sums, nin_shortcut, conv2 with the residual and the statistics of its
    output, which it returns as a second, non-differentiable output (an empty tensor when the epilogue cannot produce
    them). The backward rebuilds hn, h and h2 bit for bit: the GroupNorm apply pass with the saved mr, and conv1, whose
    stored values do not depend on the statistics epilogue. conv2 is not recomputed; its backward needs only h2, its
    weight and the incoming gradient. Then it runs the backward of conv2, nin_shortcut, norm2, conv1 and norm1 (with
    the skip gradient summed in) in the order autograd runs them without recompute, so every gradient, bias column sum
    and grad_out slot is the same.
    spec: (groups1, eps1, groups2, eps2, conv1 cache, conv2 cache, nin_shortcut cache or None)."""

    @staticmethod
    def forward(ctx, x, chsums, spec, n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb):
        require_cuda(x)
        g1, e1, g2, e2, k1, k2, ks = spec
        x = x.contiguous()
        if chsums is not None:
            hn, mr1 = gn_silu_fwd_pre(x, n1w, n1b, chsums, g1, e1, True)
        else:
            hn, mr1 = gn_silu_fwd(x, n1w, n1b, g1, e1, True)
        h, st = conv(hn, c1w, c1b, k1, "s1", want_stats=True)
        del hn
        if st is not None:
            h2, mr2 = gn_silu_fwd_pre(h, n2w, n2b, st, g2, e2, True)
        else:
            h2, mr2 = gn_silu_fwd(h, n2w, n2b, g2, e2, True)
        del h
        skip = conv(x, sw, sb, ks, "s1") if sw is not None else x
        out, stats = conv(h2, c2w, c2b, k2, "s1", residual=skip, want_stats=True)
        # the parameters go through save_for_backward so that an in-place change before the backward raises
        ctx.save_for_backward(x, mr1, mr2, n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb)
        ctx.spec = spec
        if stats is None:
            stats = torch.empty(0, device=x.device)  # "not available" marker, as ConvFn's
        ctx.mark_non_differentiable(stats)
        return out, stats

    @staticmethod
    def backward(ctx, gout, _gstats=None):
        x, mr1, mr2, n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb = ctx.saved_tensors
        inference_only(n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb)
        g1, _, g2, _, k1, k2, ks = ctx.spec
        nig = ctx.needs_input_grad
        hn = gn_silu_apply(x, n1w, n1b, mr1, True)
        h = conv(hn, c1w, c1b, k1, "s1")
        h2 = gn_silu_apply(h, n2w, n2b, mr2, True)
        # which intermediate gradients the non-recomputing graph would form
        need_hn = nig[0] or nig[3] or nig[4]  # also the skip output of norm1
        need_h = need_hn or nig[5] or nig[6]
        need_h2 = need_h or nig[7] or nig[8]
        need_res = need_hn or (sw is not None and (nig[11] or nig[12]))
        gx = gn1w = gn1b = gc1w = gc1b = gn2w = gn2b = gsw = gsb = None
        gh2, gc2w, gc2b, gskip = conv_backward(h2, c2w, gout, k2, "s1", c2b is not None, True, False, False,
                                               (need_h2, nig[9], nig[10], need_res))
        del h2
        if sw is not None and need_res:
            gskip, gsw, gsb, _ = conv_backward(x, sw, gskip, ks, "s1", sb is not None, False, False, False,
                                               (need_hn, nig[11], nig[12], False))
        if need_h2:
            gh, gn2w, gn2b = gn_silu_bwd(h, gh2, None, n2w, n2b, mr2, g2, True)
            del h, gh2
            if need_h:
                ghn, gc1w, gc1b, _ = conv_backward(hn, c1w, gh, k1, "s1", c1b is not None, False, False, False,
                                                   (need_hn, nig[5], nig[6], False))
                del hn, gh
                if need_hn:
                    gx, gn1w, gn1b = gn_silu_bwd(x, ghn, gskip, n1w, n1b, mr1, g1, True)
        grads = (gn1w, gn1b, gc1w, gc1b, gn2w, gn2b, gc2w, gc2b, gsw, gsb)
        return (gx, None, None) + tuple(g if nig[i + 3] else None for i, g in enumerate(grads))


def resnet_block_recompute(x, chsums, spec, *params):
    """-> (out, stats of out or None); see ResnetBlockRecomputeFn."""
    out, st = ResnetBlockRecomputeFn.apply(x, chsums, spec, *params)
    return out, (st if st.numel() > 0 else None)


class MaxPool2Fn(torch.autograd.Function):
    """2x2/2 max-pool of a post-ReLU activation. The backward routes dy to the first maximum of each window and gates
    it by x > 0, i.e. it returns the gradient of the *pre-activation* of the conv that produced x."""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        N, H, W, C = x.shape
        y = torch.empty(N, H // 2, W // 2, C, device=x.device, dtype=x.dtype)
        check(_L().vqb_maxpool2_fwd(ptr(x), ptr(y), N, H // 2, W // 2, C, stream_ptr()), "maxpool2_fwd")
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, gy):
        (x,) = ctx.saved_tensors
        gy = gy.contiguous()
        N, H, W, C = x.shape
        gx = torch.empty_like(x)
        check(_L().vqb_maxpool2_bwd(ptr(x), ptr(gy), 0, ptr(gx), N, H // 2, W // 2, C, 1, stream_ptr()),
              "maxpool2_bwd")
        return gx


def maxpool2(x):
    return MaxPool2Fn.apply(x)


class LpipsTailFn(torch.autograd.Function):
    """One LPIPS layer (utils.py:46-53,134-140): unit-normalise over channels, squared difference, [train mode: Dropout(0.5)
    with the counter-based mask of `seed`], 1x1 lin, spatial mean -> [N]. Gradient only w.r.t. f0 (reconstruction branch),
    gated by f0 > 0 (post-ReLU feature)."""

    @staticmethod
    def forward(ctx, f0, f1, w, seed):
        f0, f1 = f0.contiguous(), f1.contiguous()
        N, H, W, C = f0.shape
        out = torch.zeros(N, device=f0.device, dtype=torch.float32)
        wv = w.detach().reshape(-1).float().contiguous()
        if seed is None:
            check(_L().vqb_lpips_tail_fwd(ptr(f0), ptr(f1), ptr(wv), ptr(out), N, H * W, C, stream_ptr()),
                  "lpips_tail_fwd")
        else:
            check(_L().vqb_lpips_tail_fwd_dropout(ptr(f0), ptr(f1), ptr(wv), ptr(out), N, H * W, C, seed, stream_ptr()),
                  "lpips_tail_fwd_dropout")
        ctx.save_for_backward(f0, f1, wv)
        ctx.seed = seed
        return out

    @staticmethod
    def backward(ctx, g):
        f0, f1, wv = ctx.saved_tensors
        N, H, W, C = f0.shape
        g = g.float().contiguous()
        df0 = torch.empty_like(f0)
        if ctx.seed is None:
            check(_L().vqb_lpips_tail_bwd(ptr(f0), ptr(f1), ptr(wv), ptr(g), ptr(df0), N, H * W, C, stream_ptr()),
                  "lpips_tail_bwd")
        else:
            check(_L().vqb_lpips_tail_bwd_dropout(ptr(f0), ptr(f1), ptr(wv), ptr(g), ptr(df0), N, H * W, C, ctx.seed,
                                                  stream_ptr()), "lpips_tail_bwd_dropout")
        return df0, None, None, None


def lpips_tail(f0, f1, w, dropout_seed=None):
    return LpipsTailFn.apply(f0, f1, w, dropout_seed)


def lpips_dropout_mask(seed: int, N: int, HW: int, C: int, device) -> torch.Tensor:
    """The keep mask ([N, HW, C] uint8) the train-mode LPIPS tail kernels use for `seed` (parity tests)."""
    m = torch.empty(N, HW, C, device=device, dtype=torch.uint8)
    check(_L().vqb_lpips_dropout_mask(seed, N, HW, C, ptr(m), stream_ptr()), "lpips_dropout_mask")
    return m


def vq_argmin(z_flat: torch.Tensor, codebook: torch.Tensor):
    """z_flat [M, D] fp32, codebook [K, D] fp32 -> (idx int64 [M], zq fp32 [M, D], sum of squared errors (0-dim))."""
    require_cuda(z_flat)
    z_flat = z_flat.detach().float().contiguous()
    cb = codebook.detach().float().contiguous()
    M, D = z_flat.shape
    idx = torch.empty(M, device=z_flat.device, dtype=torch.int64)
    zq = torch.empty_like(z_flat)
    sq = torch.zeros((), device=z_flat.device, dtype=torch.float32)
    check(_L().vqb_vq_argmin(ptr(z_flat), ptr(cb), ptr(idx), ptr(zq), ptr(sq), M, cb.shape[0], D, stream_ptr()),
          "vq_argmin")
    return idx, zq, sq


METRICS_TILE = 32  # SSIM positions per tile side of vqb_psnr_ssim (kMTile in csrc/metrics.cu); sizes the workspace


def psnr_ssim(x: torch.Tensor, y: torch.Tensor, value_range=(0.0, 1.0)):
    """Per-item PSNR (dB) and SSIM of x against y (DESIGN.md section 7 row 25): images [B, C, H, W] -> two fp32 [B],
    clips [B, C, T, H, W] -> two fp32 [B, T], one value per frame in (b, t) order.

    x and y: contiguous CUDA tensors of one shape and dtype (float32 or bfloat16), C >= 1, H and W >= 11. Values are
    mapped to [0, 1] by value_range=(lo, hi) and clamped: (0, 1) for images, (-1, 1) for the TVAE's clips. PSNR is +inf
    for identical items. Not differentiable: inputs that require grad under grad mode are refused, so that the result
    cannot be mistaken for a loss. Every refusal raises before anything launches."""
    if not isinstance(x, torch.Tensor) or not isinstance(y, torch.Tensor):
        raise TypeError("psnr_ssim: x and y must be tensors")
    if torch.is_grad_enabled() and (x.requires_grad or y.requires_grad):
        raise RuntimeError("psnr_ssim is not differentiable: call it under torch.no_grad() or on detached tensors")
    if x.dim() not in (4, 5):
        raise ValueError(f"psnr_ssim: expected [B, C, H, W] images or [B, C, T, H, W] clips, got shape "
                         f"{tuple(x.shape)}")
    if x.shape != y.shape:
        raise ValueError(f"psnr_ssim: shapes differ: {tuple(x.shape)} vs {tuple(y.shape)}")
    if x.dtype != y.dtype or x.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"psnr_ssim: x and y must both be float32 or both bfloat16, got {x.dtype} and {y.dtype}")
    B, C = x.shape[:2]
    T = x.shape[2] if x.dim() == 5 else 1
    H, W = x.shape[-2:]
    if min(B, C, T) < 1 or H < 11 or W < 11:
        raise ValueError(f"psnr_ssim: need non-empty B, C, T and H, W >= 11 (the SSIM window), got shape "
                         f"{tuple(x.shape)}")
    try:
        lo, hi = (float(v) for v in value_range)
    except (TypeError, ValueError):
        raise ValueError(f"psnr_ssim: value_range must be a pair (lo, hi), got {value_range!r}") from None
    lo32, hi32 = (torch.tensor(v, dtype=torch.float32).item() for v in (lo, hi))  # the kernel's fp32 bounds
    if not (math.isfinite(lo32) and math.isfinite(hi32) and hi32 > lo32):
        raise ValueError(f"psnr_ssim: value_range must be finite with lo < hi in float32, got {value_range!r}")
    require_cuda(x)
    require_cuda(y)
    if x.device != y.device:
        raise ValueError(f"psnr_ssim: x is on {x.device}, y on {y.device}")
    if not (x.is_contiguous() and y.is_contiguous()):
        raise ValueError("psnr_ssim: x and y must be contiguous (the kernel reads NCHW / NCTHW in place)")
    tiles = -(-(H - 10) // METRICS_TILE) * -(-(W - 10) // METRICS_TILE)
    work = torch.empty(2 * B * T * C * tiles, device=x.device, dtype=torch.float32)
    psnr = torch.empty(B, T, device=x.device, dtype=torch.float32)
    ssim = torch.empty(B, T, device=x.device, dtype=torch.float32)
    check(_L().vqb_psnr_ssim(ptr(x), ptr(y), int(x.dtype == torch.bfloat16), B, C, T, H, W, lo32, hi32, ptr(psnr),
                             ptr(ssim), ptr(work), work.numel(), stream_ptr()), "psnr_ssim")
    if x.dim() == 4:
        return psnr.view(B), ssim.view(B)
    return psnr, ssim


# ----------------------------------------------------------------------------------------------------------------------
# Video autoencoder (tae.py): ops over NTHWC bf16 activations [N, T, H, W, Cp]. The plain functions are the no-grad
# inference path; the autograd functions after them (Conv3dFn, UpConv3dFn, AttentionHdFn, GaussReparamFn) are the
# training path that tae.py takes once a module is opted in with tae.enable_training.
def _bias_f32(bias):
    if bias is None:
        return None
    b = bias.detach()
    return b if b.dtype == torch.float32 else b.float()


def run_conv3d(g: plans.ConvGeom3d, a, wp, Cout, out, out_strides, out_off_elems=0, bias=None, res=None,
               out_f32=False):
    flags = (EPI_BIAS if bias is not None else 0) | (EPI_RES if res is not None else 0)
    dk = (Cout, tuple(out_strides), flags, out_f32)
    descs = g.__dict__.setdefault("_descs", {})
    d = descs.get(dk)
    if d is None:
        d = plans.conv3d_desc(g, Cout, out_strides, flags, out_f32)
        descs[dk] = d
    esz = out.element_size()
    check(_L().vqb_conv3d_gemm(d, ptr(a), ptr(wp), ptr(bias), (ptr(res) + out_off_elems * 2) if res is not None else 0,
                               ptr(out) + out_off_elems * esz, stream_ptr()), "conv3d_gemm")


def conv3d(x, weight, bias, cache, kind="s1", residual=None, ncthw_out=False):
    """3-D convolution of the NTHWC bf16 activation x [N, T, H, W, Cp] with an OIDHW fp32 or bf16 weight.
    kind: "s1" (3x3x3, stride 1, padding 1), "s2" (Downsample: F.pad(0,1,0,1,0,1) + 3x3x3 stride 2), "p1" (1x1x1, run
    by vqb_conv_gemm on the [N][T*H][W][C] view). residual: bf16 in the output's layout (NTHWC [N, T, H, W, Cop], or
    NCTHW with ncthw_out), summed in the epilogue. ncthw_out: write [N, Cout, T, H, W] in the weight's dtype straight
    from the epilogue (encoder z / decoder video)."""
    require_cuda(x)
    N, T, H, W, Cp = x.shape
    Cout, Cin = weight.shape[:2]
    assert Cp == plans.cpad(Cin), f"conv input has {Cp} channels, weight expects {Cin}"
    x = x.contiguous()
    b = _bias_f32(bias)
    Cop = plans.cpad(Cout)
    res = residual.contiguous() if residual is not None else None
    if kind == "p1":
        assert not ncthw_out
        g = cache.geom(("p1", N, T, H, W), lambda: plans.geom_s1(N, T * H, W, Cp, 1))
        wp = cache.get(weight, ("fwd", kind), g.tapmap, False, Cp)
        out = (torch.empty if Cop == Cout else torch.zeros)(N, T, H, W, Cop, device=x.device, dtype=torch.bfloat16)
        run_conv_gemm(g, x, wp, Cout, out, plans.nhwc_strides(T * H, W, Cop), bias=b, res=res)
        return out
    if kind == "s1":
        g = cache.geom(("s1", N, T, H, W), lambda: plans.geom3_s1(N, T, H, W, Cp))
    elif kind == "s2":
        g = cache.geom(("s2", N, T, H, W), lambda: plans.geom3_s2(N, T, H, W, Cp))
    else:
        raise ValueError(kind)
    wp = cache.get(weight, ("fwd", kind), g.tapmap, False, Cp)
    if ncthw_out:
        f32 = weight.dtype == torch.float32
        out = torch.empty(N, Cout, g.To, g.Ho, g.Wo, device=x.device, dtype=torch.float32 if f32 else torch.bfloat16)
        run_conv3d(g, x, wp, Cout, out, plans.ncthw_strides(Cout, g.To, g.Ho, g.Wo), bias=b, res=res, out_f32=f32)
        return out
    out = (torch.empty if Cop == Cout else torch.zeros)(N, g.To, g.Ho, g.Wo, Cop, device=x.device, dtype=torch.bfloat16)
    run_conv3d(g, x, wp, Cout, out, plans.nthwc_strides(g.To, g.Ho, g.Wo, Cop), bias=b, res=res)
    return out


def upsample_conv3d(x, weight, bias, cache):
    """Upsample (tae.py:110-116: nearest x2 in T, H and W, then the 3x3x3 padding-1 conv) as eight 2x2x2-tap phase
    convs over the low-resolution x (plans.geom3_up_fwd): 8/27 of the MACs, no 8x intermediate."""
    require_cuda(x)
    x = x.contiguous()
    N, t, h, w, Cp = x.shape
    Cout, Cin = weight.shape[:2]
    assert tuple(weight.shape[2:]) == (3, 3, 3) and Cp == plans.cpad(Cin)
    Cop = plans.cpad(Cout)
    out = (torch.empty if Cop == Cout else torch.zeros)(N, 2 * t, 2 * h, 2 * w, Cop, device=x.device,
                                                        dtype=torch.bfloat16)
    b = _bias_f32(bias)
    strides = plans.up3_out_strides(t, h, w, Cop)
    for pt in range(2):
        for ph in range(2):
            for pw in range(2):
                g = cache.geom(("up", N, t, h, w, pt, ph, pw), lambda: plans.geom3_up_fwd(N, t, h, w, Cp, pt, ph, pw))
                wp = cache.get(weight, ("up", pt, ph, pw), g.tapmask, False, Cp, fold=True)
                run_conv3d(g, x, wp, Cout, out, strides, out_off_elems=((pt * 2 * h + ph) * 2 * w + pw) * Cop, bias=b)
    return out


def group_norm_silu3d(x, gamma, beta, groups=32, eps=1e-6, silu=True):
    """GroupNorm(+activation) over the T*H*W voxels of an NTHWC activation (tae.py:63-71): the 2-D kernels on the
    [N][T*H][W][C] view, deterministic statistics pass. silu: an activation code (ACT_*) or a bool (swish or none)."""
    N, T, H, W, C = x.shape
    y = group_norm_silu(x.reshape(N, T * H, W, C), gamma, beta, groups, eps, silu)
    return y.view(N, T, H, W, C)


def _leaky_relu(x):
    x = x.contiguous()
    y = torch.empty_like(x)
    check(_L().vqb_leaky_relu_fwd(ptr(x), ptr(y), x.numel(), stream_ptr()), "leaky_relu_fwd")
    return y


class LeakyReLUFn(torch.autograd.Function):
    """LeakyReLU(0.2) of a bf16 NTHWC activation (vqb_leaky_relu_fwd / _bwd): the conv_in activation of
    tae_disc.PatchDiscriminator3D, which has no GroupNorm to fuse it into. The backward is gated on the saved output."""

    @staticmethod
    def forward(ctx, x):
        y = _leaky_relu(x)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, gy):
        (y,) = ctx.saved_tensors
        gy = gy.contiguous()
        dx = torch.empty_like(y)
        check(_L().vqb_leaky_relu_bwd(ptr(y), ptr(gy), ptr(dx), y.numel(), stream_ptr()), "leaky_relu_bwd")
        return dx


def leaky_relu(x):
    """LeakyReLU(0.2) of a bf16 NTHWC activation: the autograd function when grad is enabled, else one kernel."""
    require_cuda(x)
    return LeakyReLUFn.apply(x) if torch.is_grad_enabled() else _leaky_relu(x)


# head dimensions of the native attention forward and backward (vqb_attn_fwd_hd / vqb_attn_bwd_hd)
ATTN_HEAD_DIMS = tuple(range(8, 113, 8))


def attention_hd(qkv, heads, head_dim):
    """qkv [N, T, H, W, 3C] bf16 (q | k | v channel blocks) -> softmax(q k^T / sqrt(head_dim)) v as [N, T, H, W, C]
    (tae.py:26-51). head_dim a multiple of 8 from 8 to 112 (ATTN_HEAD_DIMS)."""
    return _attention_hd_fwd(qkv, heads, head_dim)[0]


def _attention_hd_fwd(qkv, heads, head_dim):
    """-> (out, lse) of attention_hd; lse [N, heads, T*H*W] is what the backward needs."""
    if head_dim not in ATTN_HEAD_DIMS:
        raise NotImplementedError(f"vqgan-training_b200: attention heads of {head_dim} channels are not supported "
                                  "(heads of 8 to 112 channels in steps of 8 only)")
    qkv = qkv.contiguous()
    N, T, H, W, C3 = qkv.shape
    C = C3 // 3
    assert C == heads * head_dim
    out = torch.empty(N, T, H, W, C, device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty(N, heads, T * H * W, device=qkv.device, dtype=torch.float32)
    check(_L().vqb_attn_fwd_hd(ptr(qkv), ptr(out), ptr(lse), N, T * H * W, C, head_dim, stream_ptr()), "attn_fwd_hd")
    return out, lse


def gauss_reparam(z, eps):
    """z [N, 2Z, ...] (mean | logvar channel halves), eps [N, Z, ...] -> mean + exp(0.5 * logvar.clamp(min=-3)) * eps
    (tae.py:259-264) in z's dtype (fp32 or bf16), computed in fp32."""
    require_cuda(z)
    check_master_dtype(z, "latent")
    z = z.contiguous()
    eps = eps.to(z.dtype).contiguous()
    N, Z2 = z.shape[:2]
    Z = Z2 // 2
    S = z[0, 0].numel()
    assert Z2 == 2 * Z and eps.shape == (N, Z) + tuple(z.shape[2:])
    out = torch.empty_like(eps)
    check(_L().vqb_gauss_reparam(ptr(z), ptr(eps), ptr(out), N, Z, S, 1 if z.dtype == torch.bfloat16 else 0,
                                 stream_ptr()), "gauss_reparam")
    return out


# ---- training path of the video autoencoder -------------------------------------------------------------------------
def _ncthw_grad_to_nthwc(gout, Cout, Cop):
    """fp32 NCTHW gradient of a module-boundary output -> bf16 NTHWC dy (vqb_nchw_to_nhwc on the [N][C][T*H][W] view)."""
    N, _, T, H, W = gout.shape
    gn = gout.float().contiguous()
    dy = torch.empty(N, T, H, W, Cop, device=gout.device, dtype=torch.bfloat16)
    check(_L().vqb_nchw_to_nhwc(ptr(gn), ptr(dy), N, Cout, T * H, W, Cop, 0, 0, stream_ptr()), "nchw_to_nhwc")
    return dy


def run_wgrad3d(g: plans.ConvGeom3d, x: torch.Tensor, dy: torch.Tensor, weight: torch.Tensor, Cout_pad: int,
                out: torch.Tensor) -> torch.Tensor:
    """OIDHW fp32 gradient (into `out`) of a 3x3x3 conv whose forward geometry is g: vqb_wgrad3d_gemm + the
    deterministic split reduction."""
    Cout, Cin = weight.shape[:2]
    descs = g.__dict__.setdefault("_descs", {})
    ent = descs.get(("wgrad3", Cout_pad))
    if ent is None:
        ksplit = choose_ksplit(g, Cout_pad)
        ent = (ksplit, plans.wgrad3d_desc(g, Cout_pad, ksplit), _L().vqb_wgrad_cols(len(g.taps), g.C))
        descs[("wgrad3", Cout_pad)] = ent
    ksplit, d, cols = ent
    partial = torch.empty(ksplit, Cout_pad, cols, device=x.device, dtype=torch.float32)
    check(_L().vqb_wgrad3d_gemm(d, ptr(dy), ptr(x), ptr(partial), stream_ptr()), "wgrad3d_gemm")
    assert out.shape == weight.shape and out.is_contiguous()
    tm = tapmap_tensor(g.tapmap, x.device)
    check(_L().vqb_wgrad_reduce(ptr(partial), ptr(out), ksplit, Cout, Cout_pad, Cin, 27, len(g.taps),
                                cols // len(g.taps), ptr(tm), 0, stream_ptr()), "wgrad_reduce")
    return out


def _bias_grad(dy, rows, Cout, Cop):
    """Bias gradient: the per-channel sums the GroupNorm backward already produced for this dy, else vqb_colsum."""
    N, T, H, W, _ = dy.shape
    gb = _take_dx_colsum(dy.view(N, T * H, W, Cop), Cop)
    if gb is None:
        gb = colsum(rows, dy, Cop)
    return gb[:Cout]


class Conv3dFn(torch.autograd.Function):
    """Autograd form of conv3d (kinds "s1", "s2", "p1"). Backward: the data gradient through the rotated 27-tap plan
    (s1), one strided conv per parity class of dx (s2, the pad plane's gradient is dropped) or the 2-D 1x1 dgrad on the
    [N][T*H][W] view (p1); the weight gradient through vqb_wgrad3d_gemm (p1: vqb_wgrad_gemm) into grad_out(weight); the
    bias gradient from the GroupNorm backward's column sums; the residual gradient is dy."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, cache, kind, ncthw_out):
        x = x.contiguous()
        out = conv3d(x, weight, bias, cache, kind, residual, ncthw_out)
        ctx.save_for_backward(x, weight)
        ctx.cache, ctx.kind, ctx.ncthw_out = cache, kind, ncthw_out
        ctx.has_bias, ctx.has_res = bias is not None, residual is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        x, weight = ctx.saved_tensors
        inference_only(weight)
        gx, gw, gb, gres = conv3d_backward(x, weight, gout, ctx.cache, ctx.kind, ctx.ncthw_out, ctx.has_bias,
                                           ctx.has_res, ctx.needs_input_grad[:4])
        return gx, gw, gb, gres, None, None, None


def conv3d_backward(x, weight, gout, cache, kind, ncthw_out, has_bias, has_res, needs):
    """Backward of conv3d(x, weight, bias, cache, kind, residual, ncthw_out) from its input x, its weight and the
    incoming gradient -> (gx, gw, gb, gres); needs: which of (x, weight, bias, residual) want a gradient."""
    N, T, H, W, Cp = x.shape
    Cout, Cin = weight.shape[:2]
    Cop = plans.cpad(Cout)
    if kind == "p1":
        g = cache.geom(("p1", N, T, H, W), lambda: plans.geom_s1(N, T * H, W, Cp, 1))
        To, Ho, Wo = T, H, W
    else:
        g = cache.geom((kind, N, T, H, W), lambda: (plans.geom3_s1 if kind == "s1" else plans.geom3_s2)(
            N, T, H, W, Cp))
        To, Ho, Wo = g.To, g.Ho, g.Wo
    dy = _ncthw_grad_to_nthwc(gout, Cout, Cop) if ncthw_out else gout.contiguous()
    gx = gw = gb = gres = None
    if needs[0]:
        gx = (torch.empty if Cp == Cin else torch.zeros)(N, T, H, W, Cp, device=x.device, dtype=torch.bfloat16)
        if kind == "p1":
            gd = cache.geom(("p1d", N, T, H, W), lambda: plans.geom_s1_dgrad(N, T * H, W, Cop, 1))
            wpd = cache.get(weight, ("dgrad", kind), gd.tapmap, True, Cop)
            run_conv_gemm(gd, dy, wpd, Cin, gx, plans.nhwc_strides(T * H, W, Cp))
        elif kind == "s1":
            gd = cache.geom(("s1d", N, T, H, W), lambda: plans.geom3_s1_dgrad(N, T, H, W, Cop))
            wpd = cache.get(weight, ("dgrad", kind), gd.tapmap, True, Cop)
            run_conv3d(gd, dy, wpd, Cin, gx, plans.nthwc_strides(T, H, W, Cp))
        else:
            for pt, ph, pw, gd in cache.geom(("s2d", N, T, H, W),
                                             lambda: plans.geom3_s2_dgrad_classes(N, T, H, W, Cop)):
                wpd = cache.get(weight, ("dgrad", kind, pt, ph, pw), gd.tapmap, True, Cop)
                strides, off = plans.s2_dgrad_out(T, H, W, Cp, pt, ph, pw)
                run_conv3d(gd, dy, wpd, Cin, gx, strides, out_off_elems=off)
    if needs[1]:
        gw = grad_out(weight)
        if kind == "p1":
            run_wgrad(g, x, dy, (Cout, Cin, 1, 1), Cop, out=gw.view(Cout, Cin, 1, 1))
        else:
            run_wgrad3d(g, x, dy, weight, Cop, gw)
    if has_bias and needs[2]:
        gb = _bias_grad(dy, N * To * Ho * Wo, Cout, Cop)
    if has_res and needs[3]:
        gres = gout if ncthw_out else dy
    return gx, gw, gb, gres


def conv3d_train(x, weight, bias, cache, kind="s1", residual=None, ncthw_out=False):
    return Conv3dFn.apply(x, weight, bias, residual, cache, kind, ncthw_out)


class ResnetBlock3dRecomputeFn(torch.autograd.Function):
    """tae.ResnetBlock as one autograd node that keeps only its input x, the two GroupNorm (mean, rstd) records and its
    parameters for the backward, instead of x, hn = swish(norm1(x)), h = conv1(hn) and h2 = swish(norm2(h)).

    The forward is the block's inference arithmetic (the kernels the non-recomputing training forward runs). The
    backward rebuilds hn, h and h2 bit for bit: the GroupNorm apply pass with the saved mr, and conv1, which is
    deterministic. conv2 is not recomputed; its backward needs only h2, its weight and the incoming gradient. Then it
    runs the backward of conv2, nin_shortcut, norm2, conv1 and norm1 (with the skip gradient summed in) in the order
    autograd runs them without recompute, so every gradient, bias column sum and grad_out slot is the same.
    spec: (groups1, eps1, groups2, eps2, conv1 cache, conv2 cache, nin_shortcut cache or None)."""

    @staticmethod
    def forward(ctx, x, spec, n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb):
        g1, e1, g2, e2, k1, k2, ks = spec
        x = x.contiguous()
        N, T, H, W, C = x.shape
        hn, mr1 = gn_silu_fwd(x.view(N, T * H, W, C), n1w, n1b, g1, e1, True)
        h = conv3d(hn.view(N, T, H, W, C), c1w, c1b, k1, "s1")
        Co = h.shape[-1]
        h2, mr2 = gn_silu_fwd(h.view(N, T * H, W, Co), n2w, n2b, g2, e2, True)
        skip = conv3d(x, sw, sb, ks, "p1") if sw is not None else x
        out = conv3d(h2.view(N, T, H, W, Co), c2w, c2b, k2, "s1", skip)
        # the parameters go through save_for_backward so that an in-place change before the backward raises
        ctx.save_for_backward(x, mr1, mr2, n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb)
        ctx.spec = spec
        return out

    @staticmethod
    def backward(ctx, gout):
        x, mr1, mr2, n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb = ctx.saved_tensors
        inference_only(n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb)
        g1, _, g2, _, k1, k2, ks = ctx.spec
        nig = ctx.needs_input_grad
        N, T, H, W, C = x.shape
        x4 = x.view(N, T * H, W, C)
        hn = gn_silu_apply(x4, n1w, n1b, mr1, True).view(N, T, H, W, C)
        h = conv3d(hn, c1w, c1b, k1, "s1")
        Co = h.shape[-1]
        h4 = h.view(N, T * H, W, Co)
        h2 = gn_silu_apply(h4, n2w, n2b, mr2, True).view(N, T, H, W, Co)
        # which intermediate gradients the non-recomputing graph would form
        need_hn = nig[0] or nig[2] or nig[3]  # also the skip output of norm1
        need_h = need_hn or nig[4] or nig[5]
        need_h2 = need_h or nig[6] or nig[7]
        need_res = need_hn or (sw is not None and (nig[10] or nig[11]))
        gx = gn1w = gn1b = gc1w = gc1b = gn2w = gn2b = gsw = gsb = None
        gh2, gc2w, gc2b, gskip = conv3d_backward(h2, c2w, gout, k2, "s1", False, c2b is not None, True,
                                                 (need_h2, nig[8], nig[9], need_res))
        del h2
        if sw is not None and need_res:
            gskip, gsw, gsb, _ = conv3d_backward(x, sw, gskip, ks, "p1", False, sb is not None, False,
                                                 (need_hn, nig[10], nig[11], False))
        if need_h2:
            gh, gn2w, gn2b = gn_silu_bwd(h4, gh2, None, n2w, n2b, mr2, g2, True)
            del h, h4, gh2
            if need_h:
                ghn, gc1w, gc1b, _ = conv3d_backward(hn, c1w, gh.view(N, T, H, W, Co), k1, "s1", False,
                                                     c1b is not None, False, (need_hn, nig[4], nig[5], False))
                del hn, gh
                if need_hn:
                    gx, gn1w, gn1b = gn_silu_bwd(x4, ghn, gskip, n1w, n1b, mr1, g1, True)
                    gx = gx.view(N, T, H, W, C)
        grads = (gn1w, gn1b, gc1w, gc1b, gn2w, gn2b, gc2w, gc2b, gsw, gsb)
        return (gx, None) + tuple(g if nig[i + 2] else None for i, g in enumerate(grads))


def resnet_block3d_recompute(x, spec, *params):
    return ResnetBlock3dRecomputeFn.apply(x, spec, *params)


class UpConv3dFn(torch.autograd.Function):
    """Autograd form of upsample_conv3d. Backward: the data gradient is one 64-tap conv over the eight parity views of dy
    (plans.geom3_up_dgrad, vqb_conv3d_dgrad_gemm: one fp32 accumulation, one rounding); the weight gradient is eight phase
    GEMMs (vqb_wgrad3d_gemm) filling one partial buffer, unfolded by vqb_wgrad_reduce_fold."""

    @staticmethod
    def forward(ctx, x, weight, bias, cache):
        x = x.contiguous()
        out = upsample_conv3d(x, weight, bias, cache)
        ctx.save_for_backward(x, weight)
        ctx.cache, ctx.has_bias = cache, bias is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        x, weight = ctx.saved_tensors
        inference_only(weight)
        cache = ctx.cache
        N, t, h, w, Cp = x.shape
        Cout, Cin = weight.shape[:2]
        Cop = plans.cpad(Cout)
        dy = gout.contiguous()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gd = cache.geom(("upd", N, t, h, w), lambda: plans.geom3_up_dgrad(N, t, h, w, Cop))
            wpd = cache.get(weight, ("updgrad",), gd.tapmask, True, Cop, fold=True)
            gx = (torch.empty if Cp == Cin else torch.zeros)(N, t, h, w, Cp, device=x.device, dtype=torch.bfloat16)
            descs = gd.__dict__.setdefault("_descs", {})
            d = descs.get(Cin)
            if d is None:
                d = descs[Cin] = plans.conv3d_dgrad_desc(gd, Cin, plans.nthwc_strides(t, h, w, Cp))
            check(_L().vqb_conv3d_dgrad_gemm(d, ptr(dy), ptr(wpd), ptr(gx), stream_ptr()), "conv3d_dgrad_gemm")
        if ctx.needs_input_grad[1]:
            C64 = ((Cp + 63) // 64) * 64
            g0 = cache.geom(("up", N, t, h, w, 0, 0, 0), lambda: plans.geom3_up_fwd(N, t, h, w, Cp, 0, 0, 0))
            ksplit = choose_ksplit(g0, Cop)
            partial = torch.empty(ksplit, Cop, 64 * C64, device=x.device, dtype=torch.float32)
            masks = []
            for pt in range(2):
                for ph in range(2):
                    for pw in range(2):
                        g = cache.geom(("up", N, t, h, w, pt, ph, pw),
                                       lambda: plans.geom3_up_fwd(N, t, h, w, Cp, pt, ph, pw))
                        descs = g.__dict__.setdefault("_descs", {})
                        d = descs.get(("upwgrad", Cop, ksplit))
                        if d is None:
                            d = descs[("upwgrad", Cop, ksplit)] = plans.wgrad3d_desc(
                                g, Cop, ksplit, dy_view=plans.up3_dy_view(N, t, h, w, Cop, pt, ph, pw),
                                ld_override=64 * C64, col_offset=(pt * 4 + ph * 2 + pw) * 8 * C64)
                        check(_L().vqb_wgrad3d_gemm(d, ptr(dy), ptr(x), ptr(partial), stream_ptr()), "wgrad3d_gemm(up)")
                        masks += g.tapmask
            gw = grad_out(weight)
            check(_L().vqb_wgrad_reduce_fold(ptr(partial), ptr(gw), ksplit, Cout, Cop, Cin, 27, 64, C64,
                                             ptr(tapmap_tensor(masks, x.device)), stream_ptr()), "wgrad_reduce_fold")
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = _bias_grad(dy, N * 8 * t * h * w, Cout, Cop)
        return gx, gw, gb, None


def upsample_conv3d_train(x, weight, bias, cache):
    return UpConv3dFn.apply(x, weight, bias, cache)


class AttentionHdFn(torch.autograd.Function):
    """Autograd form of attention_hd; the backward is vqb_attn_bwd_hd (the same head dimensions)."""

    @staticmethod
    def forward(ctx, qkv, heads, head_dim):
        qkv = qkv.contiguous()
        out, lse = _attention_hd_fwd(qkv, heads, head_dim)
        ctx.save_for_backward(qkv, out, lse)
        ctx.head_dim = head_dim
        return out

    @staticmethod
    def backward(ctx, gout):
        qkv, out, lse = ctx.saved_tensors
        N, T, H, W, C3 = qkv.shape
        dout = gout.contiguous()
        dvec = torch.empty_like(lse)
        dqkv = torch.empty_like(qkv)
        check(_L().vqb_attn_bwd_hd(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dvec), ptr(dqkv), N, T * H * W, C3 // 3,
                                   ctx.head_dim, stream_ptr()), "attn_bwd_hd")
        return dqkv, None, None


def attention_hd_train(qkv, heads, head_dim):
    return AttentionHdFn.apply(qkv, heads, head_dim)


class GaussReparamFn(torch.autograd.Function):
    """Autograd form of gauss_reparam for fp32 latents; the backward is vqb_gauss_reparam_bwd (eps carries no
    gradient: it is drawn noise)."""

    @staticmethod
    def forward(ctx, z, eps):
        z = z.contiguous()
        eps = eps.to(z.dtype).contiguous()
        ctx.save_for_backward(z, eps)
        return gauss_reparam(z, eps)

    @staticmethod
    def backward(ctx, g):
        z, eps = ctx.saved_tensors
        inference_only(z)
        N, Z2 = z.shape[:2]
        g = g.float().contiguous()
        dz = torch.empty_like(z)
        check(_L().vqb_gauss_reparam_bwd(ptr(g), ptr(z), ptr(eps), ptr(dz), N, Z2 // 2,
                                         z[0, 0].numel(), stream_ptr()), "gauss_reparam_bwd")
        return dz, None


def gauss_reparam_train(z, eps):
    return GaussReparamFn.apply(z, eps)
