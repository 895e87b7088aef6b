"""Weight-EMA oracle: the update-count schedule and the fp64 recurrence. TEST INFRASTRUCTURE (see oracle/__init__.py).

PARITY UNPINNED BY THE REFERENCE: cloneofsimo/vqgan-training keeps no moving average of the weights. This file restates
the definition of DESIGN.md section 7 row 26, the latent-diffusion EMA with its update-count warm-up, for one optimizer:

    e_0   = the parameters when the average is created (after the data-parallel constructor broadcast)
    n     = updates applied so far, 0 at creation; each AdamW launch increments it BEFORE use (the first update has n = 1)
    d_n   = min(ema_decay, (1 + n) / (10 + n))
    r_n   = 1 - d_n, in float64, rounded once to float32 (what the kernel reads)
    e_n   = e_{n-1} - r_n (e_{n-1} - p_n),  p_n the parameters AdamW has just written

Every element of the flat buffer is updated, including chunks that got no gradient (their p_n = p_{n-1}) and the zero
pads. A step that finds no gradient launches nothing and does not update. 0 < ema_decay < 1, else ValueError.
"""
from __future__ import annotations

import numpy as np


def check_decay(ema_decay) -> float:
    d = float(ema_decay)
    if not 0.0 < d < 1.0:
        raise ValueError(f"ema_decay must satisfy 0 < ema_decay < 1, got {ema_decay!r}")
    return d


def decay_at(n: int, ema_decay: float) -> float:
    """d_n (float64), n >= 1."""
    if n < 1:
        raise ValueError(f"the first update has n = 1, got n = {n}")
    return min(float(ema_decay), (1.0 + n) / (10.0 + n))


def rate_at(n: int, ema_decay: float) -> np.float32:
    """r_n = 1 - d_n rounded once to float32."""
    return np.float32(1.0 - decay_at(n, ema_decay))


def update(e, p, rate) -> np.ndarray:
    """One update in float64 with the float32 rate: e - r (e - p)."""
    e = np.asarray(e, dtype=np.float64)
    return e - float(rate) * (e - np.asarray(p, dtype=np.float64))


def recurrence(e0, params_after_each_update, ema_decay, n0: int = 0):
    """[e_{n0+1}, e_{n0+2}, ...] in float64 from e_{n0} and the parameter snapshots p_{n0+1}, p_{n0+2}, ..."""
    out, e = [], np.asarray(e0, dtype=np.float64)
    for k, p in enumerate(params_after_each_update):
        e = update(e, p, rate_at(n0 + k + 1, ema_decay))
        out.append(e)
    return out
