"""GPU (-m gpu): the 3-D PatchGAN discriminator (tae_disc.PatchDiscriminator3D) and its place in VideoTrainer.

Kernel level (the harness of test_gpu_kernel_bounds.py: sentinel-filled outputs between guard bands, NaN-surrounded
inputs): GroupNorm forward (with and without the conv-epilogue statistics) and backward with activation code 2
(LeakyReLU(0.2)), and vqb_leaky_relu_fwd / _bwd, element-wise against float64 at ragged channel counts and voxel counts
that leave partial chunks; exactly the addressed elements are written; two runs of the forward and LeakyReLU kernels
agree bit for bit (the GroupNorm backward sums its statistics with fp32 atomics, so its second run is held to the bound).

Module level: logits, D parameter gradients and the clip gradient with D frozen against the fp32 oracle
(oracle/clip_disc_oracle.py, TF32 off) on the same weights, per tensor within 1.5x the bf16-autocast peer's cosine and
norm-ratio error plus 5e-3 (the rule of test_gpu_tae_train.py).

Step level: one VideoTrainer step with the clip discriminator (hinge + LeCam, and BCE; with and without the per-frame
D) against an fp32 oracle step, per gradient tensor within the peer's margin; ten steps against the oracle's loss curve;
two gloo ranks on one GPU keep the clip D bitwise consistent; the CLI trains with --do_clip_ganloss and checkpoints.
"""
import datetime
import hashlib
import os
import subprocess
import sys
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from helpers import cosine, seeded_sd
from oracle import clip_disc_oracle as CDO
from oracle import clip_loss_oracle as CO
from oracle import loss_oracle as LO
from oracle import lpips_oracle as LP
from oracle import seeded
from oracle import tae_oracle as TO
from test_gpu_kernel_bounds import (BITS, EPS, G32, U_BF16, Guarded, check, check_bits, check_stores, gn_fwd_truth,
                                    gn_inputs, gn_stats64, rnd)
from test_gpu_tae import SMALL, make_tvae, tf32_off

pytestmark = pytest.mark.gpu

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "vqgan-training_b200")


@pytest.fixture(scope="module", autouse=True)
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import native

    lib = native.load()
    if not lib.vqb_device_ok():
        pytest.skip("needs an sm_90 device")
    return lib


def _ok(rc, what):
    import native

    native.check(rc, what)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _leaky64(u):
    return torch.where(u > 0, u, 0.2 * u)


# ------------------------------------------------------------------------------------------------ kernel bounds
GN_CASES = [(1, 1, 64, 0), (2, 7, 32, 5), (3, 1000, 96, 0), (2, 5, 2048, 1), (1, 3 * 2 ** 16 + 5, 64, 0),
            (1, 8 * 24 * 40, 256, 1)]


@pytest.mark.parametrize("N,HW,C,ratio", GN_CASES, ids=lambda v: str(v))
def test_gn_leaky_fwd_bounds(L, N, HW, C, ratio):
    x, gamma, beta, _ = gn_inputs(N, HW, C, ratio, seed=HW + C + 7)
    X = Guarded(x.numel(), torch.bfloat16, poison="nan")
    X.body.copy_(x.reshape(-1))
    name = f"gn_leaky_fwd N={N} HW={HW} C={C} mean/std={ratio}"
    mean, var = gn_stats64(x.double(), G32)
    u64, ubound = gn_fwd_truth(x, gamma, beta, 0, mean, var)[:2]  # the pre-activation and its statistics bound
    y64 = _leaky64(u64)
    bound = U_BF16 * y64.abs() + (ubound - U_BF16 * u64.abs())  # one bf16 rounding + |leaky'| <= 1 times the stats term

    def run():
        y = Guarded(x.numel(), torch.bfloat16)
        mr = Guarded(N * G32 * 2, torch.float32)
        ws = torch.empty(N * C * 2, device=DEV, dtype=torch.float64)
        _ok(L.vqb_gn_silu_fwd(X.ptr(), y.ptr(), gamma.data_ptr(), beta.data_ptr(), mr.ptr(), ws.data_ptr(), N, HW, C,
                              G32, EPS, 2, _stream()), "gn_silu_fwd")
        torch.cuda.synchronize()
        return y, mr

    y, mr = run()
    check_stores(y, torch.arange(y.n, device=DEV), name + " stores")
    check_stores(mr, torch.arange(mr.n, device=DEV), name + " mr stores")
    check(name, y.body.view(N, HW, C), y64, bound)
    y2, mr2 = run()
    check_bits(name, y.bits(), y2.bits())
    check_bits(name + " mr", mr.bits(), mr2.bits())
    x64 = x.double()
    chs = torch.stack([x64.sum(1), (x64 * x64).sum(1)], -1).float().contiguous()
    yp = Guarded(x.numel(), torch.bfloat16)
    mrp = Guarded(N * G32 * 2, torch.float32)
    _ok(L.vqb_gn_silu_fwd_pre(X.ptr(), yp.ptr(), gamma.data_ptr(), beta.data_ptr(), mrp.ptr(), chs.data_ptr(), N, HW,
                              C, G32, EPS, 2, _stream()), "gn_silu_fwd_pre")
    torch.cuda.synchronize()
    check_stores(yp, torch.arange(yp.n, device=DEV), name + " _pre stores")
    check(name + " _pre", yp.body.view(N, HW, C), y64, bound)
    # the recompute entry point takes swish / none only
    assert L.vqb_gn_silu_apply(X.ptr(), yp.ptr(), gamma.data_ptr(), beta.data_ptr(), mrp.ptr(), N, HW, C, G32, 2,
                               _stream()) == -1


GN_BWD_CASES = [((1, 1, 64), False, True), ((2, 7, 32), True, False), ((3, 1000, 96), True, True),
                ((2, 5, 2048), False, True), ((1, 3 * 2 ** 16 + 5, 64), False, False), ((1, 8 * 24 * 40, 256), True,
                                                                                        True)]


@pytest.mark.parametrize("shape,add,colsum", GN_BWD_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_gn_leaky_bwd_bounds(L, shape, add, colsum):
    N, HW, C = shape
    x, gamma, beta, gen = gn_inputs(N, HW, C, 0.0, seed=HW + C + 11)
    dy = rnd(N, HW, C, gen=gen)
    ad = rnd(N, HW, C, gen=gen) if add else None
    mean, var = gn_stats64(x.double(), G32)
    rstd = 1 / torch.sqrt(var + EPS)
    mr = torch.stack([mean, rstd], -1).float().contiguous()
    grp = torch.arange(C, device=DEV) // (C // G32)
    mc, rc = mr[..., 0].double()[:, grp].view(N, 1, C), mr[..., 1].double()[:, grp].view(N, 1, C)
    x64, dy64, ga = x.double(), dy.double(), gamma.double()
    xh = (x64 - mc) * rc
    u = xh * ga + beta.double()
    du = torch.where(u > 0, dy64, 0.2 * dy64)
    # the kernel tests the sign of its fp32 recomputation of u: within a few fp32 ulps of 0 either slope is exact
    near0 = u.abs() <= 2.0 ** -20 * ((xh * ga).abs() + beta.double().abs() + x64.abs() * rc * ga.abs())
    edu = torch.where(near0, 0.8 * dy64.abs(), torch.zeros_like(dy64))
    cpg = C // G32

    def gmean(t):
        return t.view(N, HW, G32, cpg).mean((1, 3))[:, grp].view(N, 1, C)

    g1, g2 = gmean(ga * du), gmean(ga * du * xh)
    dx64 = rc * (ga * du - g1 - xh * g2) + (ad.double() if add else 0)
    e1, e2 = gmean(ga.abs() * edu), gmean(ga.abs() * edu * xh.abs())
    bound = U_BF16 * dx64.abs() + rc * (ga.abs() * edu + e1 + xh.abs() * e2) + \
        2.0 ** -16 * rc * ((ga * du).abs() + g1.abs() + (xh * g2).abs())
    cs64 = torch.stack([du.sum(1), (du * xh).sum(1)], -1)
    Xg = Guarded(x.numel(), torch.bfloat16, poison="nan")
    Xg.body.copy_(x.reshape(-1))
    DY = Guarded(x.numel(), torch.bfloat16, poison="nan")
    DY.body.copy_(dy.reshape(-1))
    Ag = None
    if add:
        Ag = Guarded(x.numel(), torch.bfloat16, poison="nan")
        Ag.body.copy_(ad.reshape(-1))
    name = f"gn_leaky_bwd N={N} HW={HW} C={C} add={add} colsum={colsum}"

    def run():
        dx = Guarded(x.numel(), torch.bfloat16)
        dg, db = Guarded(C, torch.float32), Guarded(C, torch.float32)
        cs_out = Guarded(C, torch.float32) if colsum else None
        ws = torch.empty(N * C * 2 + N * G32 * 2, device=DEV, dtype=torch.float32)
        _ok(L.vqb_gn_silu_bwd(Xg.ptr(), DY.ptr(), Ag.ptr() if Ag else 0, dx.ptr(), gamma.data_ptr(), beta.data_ptr(),
                              mr.data_ptr(), dg.ptr(), db.ptr(), ws.data_ptr(), N, HW, C, G32, 2,
                              cs_out.ptr() if cs_out else 0, _stream()), "gn_silu_bwd")
        torch.cuda.synchronize()
        return dx, dg, db, cs_out

    dx, dg, db, cs_out = run()
    check_stores(dx, torch.arange(dx.n, device=DEV), name + " dx stores")
    got = dx.body.view(N, HW, C)
    check(name + " dx", got, dx64, bound)
    for G_, nm, ref, w in ((db, "dbeta", cs64[..., 0].sum(0), edu), (dg, "dgamma", cs64[..., 1].sum(0),
                                                                     edu * xh.abs())):
        check_stores(G_, torch.arange(C, device=DEV), f"{name} {nm} stores")
        terms = du.abs() if nm == "dbeta" else (du * xh).abs()
        check(f"{name} {nm}", G_.body, ref, w.sum((0, 1)) + 2.0 ** -14 * terms.sum((0, 1)))
    if colsum:
        check_stores(cs_out, torch.arange(C, device=DEV), name + " dx_colsum stores")
        v = got.double()
        check(name + " dx_colsum", cs_out.body, v.sum((0, 1)), 2.0 ** -14 * v.abs().sum((0, 1)))
    # the backward sums its per-channel statistics with fp32 atomics: a second run is held to the same bound, not bits
    check(name + " dx (second run)", run()[0].body.view(N, HW, C), dx64, bound)


# voxel counts x channels: one vector, ragged channel counts (24, 40, 72) and sizes past one grid-stride sweep
LEAKY_CASES = [(1, 8), (37, 24), (1001, 40), (4099, 72), (16 * 128 * 128, 64), (8 * 24 * 40, 32)]


@pytest.mark.parametrize("V,C", LEAKY_CASES, ids=lambda v: str(v))
def test_leaky_relu_kernels_bounds(L, V, C):
    n = V * C
    gen = torch.Generator(device=DEV).manual_seed(n)
    x = rnd(n, gen=gen)
    x[:8] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, float("inf"), float("-inf"), 3.0, -3.0], device=DEV,
                         dtype=torch.bfloat16)
    dy = rnd(n, gen=gen)
    X = Guarded(n, torch.bfloat16, poison="nan")
    X.body.copy_(x)
    name = f"leaky_relu V={V} C={C}"

    def fwd():
        y = Guarded(n, torch.bfloat16)
        _ok(L.vqb_leaky_relu_fwd(X.ptr(), y.ptr(), n, _stream()), "leaky_relu_fwd")
        torch.cuda.synchronize()
        return y

    y = fwd()
    check_stores(y, torch.arange(n, device=DEV), name + " fwd stores")
    x64 = x.double()
    y64 = _leaky64(x64)
    finite = torch.isfinite(x64)
    got = y.body.double()
    assert torch.equal(got[~finite], y64[~finite]), name + ": infinities"
    check(name + " fwd", got[finite], y64[finite], U_BF16 * y64[finite].abs())  # one rounding of 0.2f x
    assert torch.equal(y.body[x > 0].view(BITS[torch.bfloat16]), x[x > 0].view(BITS[torch.bfloat16])), \
        name + ": positive inputs are not passed through exactly"
    check_bits(name + " fwd", y.bits(), fwd().bits())
    ref = torch.nn.functional.leaky_relu(x.float(), 0.2).bfloat16()
    assert torch.equal(y.body.view(BITS[torch.bfloat16]), ref.view(BITS[torch.bfloat16])), name + ": != torch"

    Y = Guarded(n, torch.bfloat16, poison="nan")
    Y.body.copy_(y.body)
    DY = Guarded(n, torch.bfloat16, poison="nan")
    DY.body.copy_(dy)

    def bwd():
        dx = Guarded(n, torch.bfloat16)
        _ok(L.vqb_leaky_relu_bwd(Y.ptr(), DY.ptr(), dx.ptr(), n, _stream()), "leaky_relu_bwd")
        torch.cuda.synchronize()
        return dx

    dx = bwd()
    check_stores(dx, torch.arange(n, device=DEV), name + " bwd stores")
    dx64 = torch.where(x64 > 0, dy.double(), 0.2 * dy.double())  # gated on x: the same set as y > 0
    check(name + " bwd", dx.body, dx64, U_BF16 * dx64.abs())
    check_bits(name + " bwd", dx.bits(), bwd().bits())
    xt = x.float().requires_grad_(True)
    torch.nn.functional.leaky_relu(xt, 0.2).backward(dy.float())
    assert torch.equal(dx.body.view(BITS[torch.bfloat16]), xt.grad.bfloat16().view(BITS[torch.bfloat16])), name


# ------------------------------------------------------------------------------------------------ module
def _disc_sd(ch, n_layers, tag):
    """Oracle initialisation with GroupNorm affines and biases perturbed (so their gradients are exercised), rounded to
    bf16 values so that both sides start from exactly the same weights."""
    torch.manual_seed(sum(map(ord, tag)))
    sd = CDO.PatchDiscriminator3D(ch=ch, n_layers=n_layers).state_dict()
    for k, v in sd.items():
        if k.endswith("norm.weight"):
            v.add_(torch.randn_like(v) * 0.2)
        elif k.endswith("bias"):
            v.add_(torch.randn_like(v) * 0.05)
    return {k: v.bfloat16().float() for k, v in sd.items()}


def _native_disc(sd, ch, n_layers):
    import tae
    import tae_disc

    m = tae_disc.PatchDiscriminator3D(ch=ch, n_layers=n_layers)
    m.load_state_dict(sd, strict=True)
    return tae.enable_training(m.cuda())


def _err(ours, truth):
    """(1 - cosine, |norm ratio - 1|)."""
    return 1 - cosine(ours, truth), abs(ours.double().norm().item() / (truth.double().norm().item() + 1e-30) - 1)


def _bar(what, ours, truth, peer):
    ec, en = _err(ours, truth)
    pc, pn = _err(peer, truth)
    print(f"  {what}: cosine err {ec:.2e} (peer {pc:.2e}), norm err {en:.2e} (peer {pn:.2e})")
    assert ec <= 1.5 * pc + 5e-3 and en <= 1.5 * pn + 5e-3, (what, ec, pc, en, pn)


MODULE_CASES = [(32, 1, (2, 8, 16, 16)), (32, 2, (1, 8, 48, 80)), (64, 3, (1, 8, 32, 32)), (64, 1, (1, 4, 24, 40)),
                (32, 3, (2, 16, 16, 24)), (64, 2, (1, 8, 48, 80))]


@pytest.mark.parametrize("ch,n_layers,shape", MODULE_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_module_against_the_oracle(ch, n_layers, shape):
    B, T, H, W = shape
    sd = _disc_sd(ch, n_layers, f"disc{ch}_{n_layers}")
    x = seeded.tensor(f"clip_disc/x{T}_{H}_{W}", (B, 3, T, H, W), 1.0, "uniform").bfloat16().float().cuda()
    m = _native_disc(sd, ch, n_layers)
    f = 2 ** n_layers
    L_ = (T // f) * (H // f) * (W // f)
    gy = seeded.tensor(f"clip_disc/gy{L_}", (B, L_)).cuda()
    with torch.no_grad():
        inf = m(x)
    logits = m(x)
    assert logits.shape == (B, L_) and torch.equal(inf, logits.detach())
    (logits * gy).sum().backward()
    ours_p = {k: p.grad for k, p in m.named_parameters()}
    m.requires_grad_(False)
    xg = x.clone().requires_grad_(True)
    (m(xg) * gy).sum().backward()

    def oracle(autocast):
        p = {k: v.cuda().clone().requires_grad_(True) for k, v in sd.items()}
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            lo = CDO.forward(p, x, n_layers).float()
        (lo * gy).sum().backward()
        xo = x.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            lx = CDO.forward({k: v.detach() for k, v in p.items()}, xo, n_layers).float()
        (lx * gy).sum().backward()
        return lo.detach(), {k: v.grad for k, v in p.items()}, xo.grad

    with tf32_off():
        tl, tp, tx = oracle(False)
    pl, pp, px = oracle(True)
    print(f"\nclip D ch={ch} n_layers={n_layers} clip {tuple(x.shape)}")
    _bar("logits", logits.detach(), tl, pl)
    _bar("clip gradient (D frozen)", xg.grad, tx, px)
    assert set(ours_p) == set(tp)
    for k in sorted(tp):
        _bar(f"d {k}", ours_p[k], tp[k], pp[k])


def test_bf16_module_is_inference_only():
    import tae_disc

    m = tae_disc.PatchDiscriminator3D(ch=32, n_layers=2).cuda().bfloat16()
    x = torch.rand(1, 3, 4, 16, 16, device=DEV) * 2 - 1
    with torch.no_grad():
        y = m(x)
    assert y.dtype == torch.bfloat16 and y.shape == (1, 16) and bool(torch.isfinite(y).all())
    with pytest.raises(RuntimeError):
        m(x)


# ------------------------------------------------------------------------------------------------ the training step
LR = 1e-4
CLIP_CH, CLIP_LAYERS = 32, 2


def _trainer(tsd, psd, dsd, disc_type, frame_d):
    import tae
    import tae_disc
    import tae_trainer
    import utils

    m = tae.TVAE(**SMALL.kwargs())
    m.load_state_dict(tsd)
    pd = None
    if frame_d:
        pd = utils.PatchDiscriminator()
        pd.load_state_dict(psd, strict=True)
        pd = pd.cuda()
    d3 = tae_disc.PatchDiscriminator3D(ch=CLIP_CH, n_layers=CLIP_LAYERS)
    d3.load_state_dict(dsd, strict=True)
    return tae_trainer.VideoTrainer(m.cuda(), None, pd, disc_type=disc_type, use_lecam=disc_type == "hinge",
                                    lr_vae=LR, lr_disc=LR, clip_discriminator=d3.cuda(), lr_clip_disc=LR)


class OracleStep:
    """The same step in the oracle's autograd (MSE reconstruction, per-frame D optional, clip D), fp32 or under bf16
    autocast (the peer), with torch.optim.AdamW."""

    def __init__(self, tsd, psd, dsd, disc_type, frame_d, autocast):
        kw = dict(weight_decay=1e-3, betas=(0.9, 0.95))
        self.tp = {k: v.cuda().clone().requires_grad_(True) for k, v in tsd.items()}
        self.dp = {k: v.cuda().clone().requires_grad_("scaling_layer" not in k) for k, v in psd.items()}
        self.cp = {k: v.cuda().clone().requires_grad_(True) for k, v in dsd.items()}
        self.opt_g = torch.optim.AdamW(self.tp.values(), lr=LR, **kw)
        self.opt_d = torch.optim.AdamW([v for v in self.dp.values() if v.requires_grad], lr=LR, **kw)
        self.opt_c = torch.optim.AdamW(self.cp.values(), lr=LR, **kw)
        self.anchors, self.canchors = [0.0, 0.0], [0.0, 0.0]
        self.disc_type, self.frame_d, self.autocast = disc_type, frame_d, autocast

    def _d_step(self, fwd, params, opt, anchors, real_in, fake_in):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.autocast):
            real, fake = fwd(params, real_in).float(), fwd(params, fake_in).float()
        loss, ar, af, _ = LO.gan_disc_loss(real, fake, self.disc_type)
        anchors[:] = [0.9 * anchors[0] + 0.1 * ar, 0.9 * anchors[1] + 0.1 * af]
        if self.disc_type == "hinge":
            loss = loss + 0.1 * LO.lecam_loss(real, fake, anchors[0], anchors[1])
        opt.zero_grad()
        loss.backward()
        grads = {k: v.grad.float().clone() for k, v in params.items() if v.requires_grad}
        opt.step()
        return grads

    def _g(self, fwd, params, x):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.autocast):
            fake = fwd({k: v.detach() for k, v in params.items()}, x).float()
        if self.disc_type == "bce":
            return F.binary_cross_entropy_with_logits(fake, torch.ones_like(fake))
        return -fake.mean()

    def step(self, x, eps):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.autocast):
            decz, z = TO.forward(self.tp, x, eps, SMALL)
        decz, z = decz.float(), z.float()
        patchd = lambda p, v: CO.patchd_clip(p, v)  # noqa: E731
        clipd = lambda p, v: CDO.forward(p, v, CLIP_LAYERS)  # noqa: E731
        dgrads = self._d_step(patchd, self.dp, self.opt_d, self.anchors, x, decz.detach()) if self.frame_d else {}
        cgrads = self._d_step(clipd, self.cp, self.opt_c, self.canchors, x, decz.detach())
        loss = F.mse_loss(decz, x) + LO.vae_loss_function(x, decz, z)[0]
        if self.frame_d:
            loss = loss + self._g(patchd, self.dp, LO.gradnorm(decz, 1.0))
        loss = loss + self._g(clipd, self.cp, LO.gradnorm(decz, 1.0))
        self.opt_g.zero_grad()
        loss.backward()
        tgrads = {k: v.grad.float().clone() for k, v in self.tp.items()}
        self.opt_g.step()
        return loss.item(), tgrads, dgrads, cgrads


def _weights():
    _, tsd = make_tvae(SMALL, "tae_small", torch.float32)
    psd = seeded_sd(LP.patchd_state_dict_shapes(), "patchd")
    dsd = _disc_sd(CLIP_CH, CLIP_LAYERS, "step")
    return tsd, psd, dsd


def _eps(seed, z):
    torch.manual_seed(seed)
    return torch.randn_like(z.chunk(2, dim=1)[0])


def _cos_check(what, ours, truth, peer):
    keys = sorted(truth)
    ref = np.array([truth[k].norm().item() for k in keys])
    big = ref > 1e-3 * ref.max()
    cos = np.array([cosine(ours[k], truth[k]) for k in keys])[big]
    pcos = np.array([cosine(peer[k], truth[k]) for k in keys])[big]
    print(f"\n{what}: {big.sum()} tensors, cosine min {cos.min():.5f} (peer {pcos.min():.5f})")
    bad = [(k, round(c, 5), round(pc, 5)) for k, c, pc in zip(np.array(keys)[big], cos, pcos)
           if 1 - c > 1.5 * (1 - pc) + 5e-3]
    assert not bad, bad


@pytest.mark.parametrize("disc_type,frame_d", [("hinge", False), ("hinge", True), ("bce", False), ("bce", True)])
def test_one_step_matches_oracle_autograd(disc_type, frame_d):
    tsd, psd, dsd = _weights()
    tr = _trainer(tsd, psd, dsd, disc_type, frame_d)
    x = seeded.tensor("clip_gpu/train_x", (1, 3, 4, 32, 32), 1.0, "uniform").bfloat16().float().cuda()
    torch.manual_seed(3)
    out = tr.step(x)
    for k in ("clip_d_loss", "clip_g_gan_loss", "clip_disc_acc", "clip_lecam_loss", "clip_avg_real_logits",
              "clip_avg_fake_logits"):
        assert k in out, k
    assert ("d_loss" in out) == frame_d
    eps = _eps(3, out["z"])
    ours_t = {k: p.grad for k, p in tr.vae.named_parameters()}
    ours_c = {k: p.grad for k, p in tr.clip_disc.named_parameters()}
    with tf32_off():
        tl, tt, td, tc = OracleStep(tsd, psd, dsd, disc_type, frame_d, False).step(x, eps)
    pl, pt, pdg, pc = OracleStep(tsd, psd, dsd, disc_type, frame_d, True).step(x, eps)
    ol = out["overall_vae_loss"].item()
    print(f"\nloss ours {ol:.6f} fp32 oracle {tl:.6f} peer {pl:.6f}")
    assert abs(ol - tl) <= 1.5 * abs(pl - tl) + 2e-3 * abs(tl) + 1e-4
    assert set(ours_c) == set(tc)
    _cos_check("TVAE parameter gradients", ours_t, tt, pt)
    _cos_check("clip D parameter gradients", ours_c, tc, pc)
    if frame_d:
        _cos_check("PatchD parameter gradients", {k: p.grad for k, p in tr.disc.named_parameters()}, td, pdg)


def test_ten_steps_track_the_oracle_loss_curve():
    tsd, psd, dsd = _weights()
    tr = _trainer(tsd, psd, dsd, "bce", False)
    x = seeded.tensor("clip_gpu/train_x", (1, 3, 4, 32, 32), 1.0, "uniform").bfloat16().float().cuda()
    ours, epss = [], []
    for i in range(10):
        torch.manual_seed(100 + i)
        out = tr.step(x)
        ours.append(out["overall_vae_loss"].item())
        epss.append(_eps(100 + i, out["z"]))

    def curve(autocast):
        o = OracleStep(tsd, psd, dsd, "bce", False, autocast)
        return np.array([o.step(x, e)[0] for e in epss])

    with tf32_off():
        truth = curve(False)
    peer = curve(True)
    ours = np.array(ours)
    e, pe = np.abs(ours - truth) / np.abs(truth), np.abs(peer - truth) / np.abs(truth)
    print("\nloss curve ours", ours, "\nfp32", truth, "\npeer", peer, f"\nmax rel dev ours {e.max():.3e} peer "
          f"{pe.max():.3e}")
    assert e[0] < 1e-2 and e.max() <= 1.5 * pe.max() + 2e-2


# ------------------------------------------------------------------------------------------------ data parallel
def _digest(tensors):
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def _ddp_worker(rank, world, port, out, q):
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), VQB_OFFLINE="1")
    os.environ.pop("VQB_DDP_OVERLAP", None)
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
        tsd, psd, dsd = _weights()
        tr = _trainer(tsd, psd, dsd, "hinge", False)
        store = tr.optimizer_clip_D.store
        log = []
        reduce = tr._clip_disc_dp.allreduce_grads

        def snooped():
            store.collect()
            log.append(store.grads.detach().clone())
            reduce()
            log.append(store.grads.detach().clone())

        tr._clip_disc_dp.allreduce_grads = snooped
        torch.manual_seed(30 + rank)
        steps = []
        for i in range(3):
            x = seeded.tensor(f"video_ddp/x{rank}_{i}", (1, 3, 4, 32, 32), 1.0, "uniform").bfloat16().float().cuda()
            tr.step(x)
            o = tr.optimizer_clip_D
            steps.append({"w": _digest([o.store.params]), "m": _digest([o.exp_avg, o.exp_avg_sq]),
                          "a": _digest([tr.clip_lecam_anchor_real_logits, tr.clip_lecam_anchor_fake_logits]),
                          "tvae": _digest([tr.optimizer_G.store.params])})
        torch.save({"local": log[0].cpu(), "reduced": log[1].cpu()}, os.path.join(out, f"clip_d_{rank}.pt"))
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok", steps))
    except BaseException:
        q.put((rank, "error", traceback.format_exc()))
        raise


def test_two_gloo_ranks_keep_the_clip_disc_consistent(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31100 + (os.getpid() % 500)
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=900) for _ in procs]
    finally:
        for p in procs:
            p.join(120)
            if p.is_alive():
                p.terminate()
                p.join(30)
    errors = [r[2] for r in res if r[1] == "error"]
    assert not errors, "\n".join(errors)
    s0, s1 = [r[2] for r in sorted(res, key=lambda r: r[0])]
    assert s0 == s1, "clip D weights, AdamW moments, anchors or TVAE weights differ between ranks"
    a, b = torch.load(tmp_path / "clip_d_0.pt"), torch.load(tmp_path / "clip_d_1.pt")
    assert torch.equal(a["reduced"], b["reduced"])
    assert not torch.equal(a["local"], b["local"]), "the ranks' local gradients are equal (the check is vacuous)"
    mean = (a["local"].double() + b["local"].double()) / 2
    err = (a["reduced"].double() - mean).abs()
    assert bool((err <= 2.0 ** -23 * mean.abs() + 1e-38).all()), "the all-reduced gradient is not the rank mean"


# ------------------------------------------------------------------------------------------------ entry point
def test_cli_trains_with_the_clip_disc_and_saves(tmp_path):
    import tae

    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR",
                                                            "MASTER_PORT")}
    env["VQB_OFFLINE"] = "1"
    args = ["--vae_ch", "32", "--vae_ch_mult", "1,8", "--vae_num_res_blocks", "1", "--vae_z_channels", "4",
            "--clip_frames", "4", "--resolution", "32", "--batch_size", "1", "--no_lpips", "--do_clip_ganloss",
            "--clip_disc_ch", "32", "--clip_disc_layers", "2", "--disc_type", "hinge", "--use_lecam", "True",
            "--max_steps", "3", "--evaluate_every_n_steps", "3", "--run_name", "clipd"]
    p = subprocess.run([sys.executable, os.path.join(PKG, "tae_trainer.py")] + args, cwd=tmp_path, env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "clip_d_loss" in p.stderr and "clip_lecam_loss" in p.stderr, p.stderr
    ck = torch.load(tmp_path / "ckpt" / "clipd" / "tvae_step_3.pt")
    m = tae.TVAE(**SMALL.kwargs() | {"resolution": 32})
    m.load_state_dict(ck, strict=True)
    assert all(torch.isfinite(v).all() for v in ck.values())
