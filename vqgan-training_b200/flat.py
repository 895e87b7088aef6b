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
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List

import torch

import native
import ops

CHUNK = 1024


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
    at `step()` are skipped exactly like torch does."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=1e-2):
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
    def upload_hyper(self, active=None):
        if self._rec_dev is None:
            dev = self.store.params.device
            self._rec_dev = torch.zeros(28, device=dev, dtype=torch.float32)
            self._rec_pin = [torch.zeros(28, dtype=torch.float32).pin_memory() for _ in range(4)]
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
        self._rec_dev.copy_(self._rec_pin[i], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._rec_ev[i] = ev

    def launch(self, active, pack=False):
        tab = self._chunk_table(active)
        native.check(native.load().vqb_adamw_flat_dev(
            self.store.params.data_ptr(), self.store.grads.data_ptr(), self.exp_avg.data_ptr(),
            self.exp_avg_sq.data_ptr(), tab.data_ptr(), self.store.total // CHUNK, self._rec_dev.data_ptr(),
            C.c_float(self.grad_scale), native.stream_ptr()), "adamw_flat_dev")
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
