"""Flat parameter / gradient / optimizer-state storage for the training step and the fused AdamW over it.

Why: the reference's optimizer step is `optim.AdamW([two lr groups], weight_decay=1e-3, betas=(0.9, 0.95))` plus a
cosine-with-warmup schedule (vae_trainer.py:455-475,486-490) over ~250 tensors, and its (intended) gradient all-reduce is
DDP's bucketed copy-in / all-reduce / copy-out. Here every trainable tensor of a model lives in ONE fp32 buffer:

  * `param.data` of every parameter is a view into `FlatParams.params` (state_dict keys/shapes unchanged);
  * weight-gradient kernels write straight into the matching slot of `FlatParams.grads` (ops.grad_out), autograd adopts
    that view as `param.grad` — so the NCCL all-reduce runs on `grads` in place (no copy-in/copy-out passes) and
  * `FlatAdamW.step()` is one kernel (vqb_adamw_flat) over (params, grads, exp_avg, exp_avg_sq), followed by one
    vqb_pack_weights_multi launch that refreshes every cached bf16 GEMM operand.

Each tensor's slot is padded to a multiple of 1024 elements (the kernel's chunk); pad elements stay zero.

`FlatAdamW(..., ema_decay=d)` also keeps an exponential moving average of the parameters in a flat fp32 buffer `ema`,
updated by the same kernel launch (vqb_adamw_ema_flat_dev) with the update-count warm-up of latent diffusion's EMA:
the n-th update (n = 1, 2, ...) uses d_n = min(d, (1 + n) / (10 + n)). `averaged_copy(module)` builds an inference module
over that buffer.
"""
from __future__ import annotations

import copy
import ctypes as C
from typing import Iterable, List

import torch

import native
import ops

CHUNK = 1024
RECORD_FLOATS = 28  # the AdamW hyper-parameter record of vqb_adamw_fill_record; the EMA rate follows it


def check_ema_decay(ema_decay) -> float:
    """0 < ema_decay < 1 (a float), else ValueError."""
    try:
        d = float(ema_decay)
    except (TypeError, ValueError):
        raise ValueError(f"ema_decay must be a number in (0, 1), got {ema_decay!r}") from None
    if not 0.0 < d < 1.0:
        raise ValueError(f"ema_decay must satisfy 0 < ema_decay < 1, got {ema_decay!r}")
    return d


def ema_decay_at(n: int, ema_decay: float) -> float:
    """d_n of the n-th EMA update (n >= 1): min(ema_decay, (1 + n) / (10 + n)), in double."""
    return min(ema_decay, (1.0 + n) / (10.0 + n))


def ema_rate(n: int, ema_decay: float) -> float:
    """The kernel's rate of the n-th update: 1 - d_n in double, rounded once to fp32."""
    return float(torch.tensor(1.0 - ema_decay_at(n, ema_decay), dtype=torch.float32))


class FlatParams:
    """Re-homes the trainable parameters of `module` into one flat fp32 buffer (+ a same-shaped gradient buffer)."""

    def __init__(self, params: Iterable[torch.nn.Parameter]):
        self.plist: List[torch.nn.Parameter] = [p for p in params if p.requires_grad]
        if not self.plist:
            raise ValueError("FlatParams: no trainable parameters")
        dev = self.plist[0].device  # (a CPU store is plain storage for the gloo host-logic tests; kernels need CUDA)
        self.offsets, off = [], 0
        for p in self.plist:
            if p.dtype != torch.float32:
                raise RuntimeError("FlatParams: master parameters must be fp32")
            self.offsets.append(off)
            off += -(-p.numel() // CHUNK) * CHUNK
        self.total = off
        self.params = torch.zeros(off, device=dev, dtype=torch.float32)
        self.grads = torch.zeros(off, device=dev, dtype=torch.float32)
        with torch.no_grad():
            for p, o in zip(self.plist, self.offsets):
                v = self.params[o:o + p.numel()].view(p.shape)
                v.copy_(p.data)
                p.data = v
        self._slot_ptr = [self.grads.data_ptr() + 4 * o for o in self.offsets]
        self._handed_out = set()
        for i, p in enumerate(self.plist):
            ops.register_grad_slot(p, self, i)
        ops.weights_updated(self.plist)  # data_ptr of every master weight moved

    # ------------------------------------------------------------------ gradient slots
    def slot(self, i: int) -> torch.Tensor:
        """A FRESH view of parameter i's gradient slot (fresh so that autograd may adopt it as `.grad` without a copy)."""
        p, o = self.plist[i], self.offsets[i]
        return self.grads[o:o + p.numel()].view(p.shape)

    def take_slot(self, i: int):
        """First gradient contribution of parameter i in this accumulation window -> its slot view; later ones -> None
        (the caller allocates a temporary and autograd accumulates it into the slot in place)."""
        if i in self._handed_out:
            return None
        self._handed_out.add(i)
        return self.slot(i)

    def zero_grad(self):
        for p in self.plist:
            p.grad = None
        self._handed_out.clear()

    @torch.no_grad()
    def collect(self, indices=None):
        """After backward: make every existing `.grad` (of the parameters `indices`, default all) live in its slot —
        copies only gradients produced elsewhere, e.g. bias sums — and return the 'has a gradient' flags."""
        stray_dst, stray_src, active = [], [], []
        for i in (range(len(self.plist)) if indices is None else indices):
            p = self.plist[i]
            g = p.grad
            if g is None:
                active.append(False)
                continue
            active.append(True)
            if g.data_ptr() != self._slot_ptr[i] or not g.is_contiguous() or g.dtype != torch.float32:
                s = self.slot(i)
                stray_dst.append(s)
                stray_src.append(g)
                p.grad = s
                self._handed_out.add(i)
        if stray_dst:
            torch._foreach_copy_(stray_dst, stray_src)
        return tuple(active)


class FlatAdamW(torch.optim.Optimizer):
    """torch.optim.AdamW semantics (decoupled weight decay, bias correction) as ONE kernel over a FlatParams store.

    `params` is the usual list of parameter groups (each with its own lr — the two groups of vae_trainer.py:455-465);
    lr schedulers (LambdaLR cosine, :486-490) act on `param_groups[i]["lr"]` as usual. Parameters whose `.grad` is None
    at `step()` are skipped exactly like torch does.

    ema_decay=None: no moving average. With 0 < ema_decay < 1 the optimizer also owns `ema`, a flat fp32 copy of
    `store.params` taken here, and `ema_updates`, the count n of updates applied to it. Every launch of the AdamW kernel
    (`step()` with at least one gradient, or `upload_hyper()` + `launch()`) then performs one update after AdamW has
    written the parameters: n += 1, ema -= (1 - d_n) (ema - params) over the whole buffer (tensors without a gradient
    and the zero pads included), 1 - d_n computed in double and rounded once to fp32. `reset_ema()` restarts it."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=1e-2, ema_decay=None):
        if ema_decay is not None:  # before anything is allocated
            ema_decay = check_ema_decay(ema_decay)
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        if len(self.param_groups) > 4:
            raise ValueError("FlatAdamW supports at most 4 parameter groups")
        ordered = [p for g in self.param_groups for p in g["params"]]
        self.store = FlatParams(ordered)
        if len(self.store.plist) != len(ordered):
            raise ValueError("FlatAdamW: every parameter must require grad")
        n = self.store.total
        dev = self.store.params.device
        self.exp_avg = torch.zeros(n, device=dev, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(n, device=dev, dtype=torch.float32)
        self._group_of = []
        for gi, g in enumerate(self.param_groups):
            self._group_of += [gi] * len(g["params"])
            g.setdefault("step", 0)
        for p, o in zip(self.store.plist, self.store.offsets):  # torch-style per-parameter state views (checkpointing)
            self.state[p] = {"exp_avg": self.exp_avg[o:o + p.numel()].view(p.shape),
                             "exp_avg_sq": self.exp_avg_sq[o:o + p.numel()].view(p.shape)}
        self._chunk_tables = {}
        self.grad_scale = 1.0
        self._rec_dev = None
        self.ema_decay = ema_decay
        self.ema = None
        self.ema_updates = 0
        self.ema_generation = 0  # bumped whenever `ema` may have been written (an update or a reset): packs re-check it
        if ema_decay is not None:
            self.ema = self.store.params.clone()

    @torch.no_grad()
    def reset_ema(self):
        """Restarts the average from the current parameters (the update count returns to 0)."""
        if self.ema is None:
            raise RuntimeError("FlatAdamW.reset_ema: this optimizer keeps no EMA (ema_decay=None)")
        self.ema.copy_(self.store.params)
        self.ema_updates = 0
        self.ema_generation += 1

    def averaged_copy(self, module: torch.nn.Module) -> torch.nn.Module:
        """An inference module of `module`'s class over the averaged weights.

        Every parameter of `module` that lives in this optimizer's store becomes, in the copy, a view into `ema`
        (requires_grad=False; no copy); frozen parameters and buffers are copied. Each conv of the copy has its own
        bf16 pack cache. The first forward of any submodule of the copy after the average moved re-packs them; the
        training step never does. The copy's state_dict has `module`'s keys."""
        if self.ema is None:
            raise RuntimeError("FlatAdamW.averaged_copy: this optimizer keeps no EMA (ema_decay=None)")
        slot = {id(p): (p, o) for p, o in zip(self.store.plist, self.store.offsets)}
        memo, averaged = {}, []
        for m in module.modules():
            pc = getattr(m, "_packed", None)
            if isinstance(pc, ops.PackedCache):
                memo[id(pc)] = ops.PackedCache()
        for p in module.parameters():
            hit = slot.get(id(p))
            if hit is not None and id(p) not in memo:
                o = hit[1]
                q = torch.nn.Parameter(self.ema[o:o + p.numel()].view(p.shape), requires_grad=False)
                memo[id(p)] = q
                averaged.append(q)
        if not averaged:
            raise ValueError("FlatAdamW.averaged_copy: no parameter of the module lives in this optimizer")
        out = copy.deepcopy(module, memo)
        seen = [None]

        def refresh(_mod, _args):  # forward pre-hook of every submodule: some pack through a child's cache directly
            if seen[0] != self.ema_generation:
                ops.weights_updated(averaged)  # only the copy's pack entries live at these addresses
                seen[0] = self.ema_generation

        for m in out.modules():
            m.register_forward_pre_hook(refresh)
        return out

    def _chunk_table(self, active):
        t = self._chunk_tables.get(active)
        if t is None:
            import numpy as np

            tab = np.full(self.store.total // CHUNK, 255, dtype=np.uint8)
            for i, (p, o) in enumerate(zip(self.store.plist, self.store.offsets)):
                if active[i]:
                    tab[o // CHUNK:(o + -(-p.numel() // CHUNK) * CHUNK) // CHUNK] = self._group_of[i]
            t = torch.from_numpy(tab).to(self.store.params.device)
            if len(self._chunk_tables) > 16:
                self._chunk_tables.clear()
            self._chunk_tables[active] = t
        return t

    def zero_grad(self, set_to_none: bool = True):
        self.store.zero_grad()

    # The step is split so that a captured CUDA graph can contain the kernel while the host still drives the schedule:
    #   upload_hyper()  host: advance the step counts, compute lr / bias corrections, copy the 28-float record to the
    #                   device (pinned ring buffer, stream-ordered) — runs BEFORE a graph replay
    #   launch()        device: vqb_adamw_flat_dev (+ the re-pack of the bf16 operands when pack=True) — capturable
    #                   (+ with an EMA: advance its count and append 1 - d_n to the record as float 28)
    def upload_hyper(self, active=None):
        if self._rec_dev is None:
            dev = self.store.params.device
            nrec = RECORD_FLOATS + (1 if self.ema is not None else 0)
            self._rec_dev = torch.zeros(nrec, device=dev, dtype=torch.float32)
            self._rec_pin = [torch.zeros(nrec, dtype=torch.float32).pin_memory() for _ in range(4)]
            self._rec_ev = [None] * 4
            self._rec_i = 0
        groups = (native.VqbAdamwGroup * len(self.param_groups))()
        for gi, g in enumerate(self.param_groups):
            if active is None or any(active[i] for i in range(len(active)) if self._group_of[i] == gi):
                g["step"] += 1
            b1, b2 = g["betas"]
            groups[gi] = native.VqbAdamwGroup(lr=float(g["lr"]), beta1=float(b1), beta2=float(b2), eps=float(g["eps"]),
                                              weight_decay=float(g["weight_decay"]), step=max(1, int(g["step"])))
        i = self._rec_i
        self._rec_i = (i + 1) % len(self._rec_pin)
        if self._rec_ev[i] is not None:
            self._rec_ev[i].synchronize()  # the copy that last read this pinned slot (4 steps ago) has executed
        native.check(native.load().vqb_adamw_fill_record(len(self.param_groups), groups, self._rec_pin[i].data_ptr()),
                     "adamw_fill_record")
        if self.ema is not None:
            n = self.ema_updates + 1
            self._rec_pin[i][RECORD_FLOATS] = ema_rate(n, self.ema_decay)
            self.ema_updates = n
            self.ema_generation += 1
        self._rec_dev.copy_(self._rec_pin[i], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._rec_ev[i] = ev

    def launch(self, active, pack=False):
        tab = self._chunk_table(active)
        if self.ema is None:
            native.check(native.load().vqb_adamw_flat_dev(
                self.store.params.data_ptr(), self.store.grads.data_ptr(), self.exp_avg.data_ptr(),
                self.exp_avg_sq.data_ptr(), tab.data_ptr(), self.store.total // CHUNK, self._rec_dev.data_ptr(),
                C.c_float(self.grad_scale), native.stream_ptr()), "adamw_flat_dev")
        else:
            native.check(native.load().vqb_adamw_ema_flat_dev(
                self.store.params.data_ptr(), self.store.grads.data_ptr(), self.exp_avg.data_ptr(),
                self.exp_avg_sq.data_ptr(), self.ema.data_ptr(), tab.data_ptr(), self.store.total // CHUNK,
                self._rec_dev.data_ptr(), self._rec_dev.data_ptr() + 4 * RECORD_FLOATS, C.c_float(self.grad_scale),
                native.stream_ptr()), "adamw_ema_flat_dev")
            self.ema_generation += 1
        if pack:
            ops.weights_updated(self.store.plist)

    @torch.no_grad()
    def step(self, closure=None):
        if not self.store.params.is_cuda:
            raise RuntimeError("FlatAdamW.step: the fused optimizer kernel runs on sm_90a only (no CPU fallback)")
        active = self.store.collect()
        if not any(active):
            return None
        self.upload_hyper(active)
        self.launch(active)
        # the global optimizer post-step hook (ops._optimizer_post_step) re-packs the bf16 operands of these weights
        return None
