"""GPU (-m gpu): per-frame LPIPS / PatchGAN on [B, 3, T, H, W] clips and the video training step (tae_trainer).

Kernel level (the harness of test_gpu_kernel_bounds.py: sentinel-filled outputs between guard bands, NaN-surrounded
inputs): the clip boundary kernels are bit-identical to the 2-D kernels applied to the ATen-folded frames (forward) and
to the 2-D backward followed by an ATen scatter into a zero clip (backward).

Module level: LPIPS and PatchDiscriminator on a clip equal the same modules on the folded frames, forward and clip
gradient. LPIPS sums each layer's spatial mean with fp32 atomics, so its forward is compared to a few ulps; everything
else is compared bit for bit.

Step level: one VideoTrainer.step against fp32 oracle autograd (tae_oracle + clip_loss_oracle + loss_oracle, TF32 off)
on the same weights, held per tensor to 1.5x the bf16-autocast peer's cosine error plus 5e-3 (the rule of
test_gpu_tae_train.py); ten steps against the oracle's loss curve; recompute=True against the plain path.
"""
import numpy as np
import pytest
import torch

from helpers import cosine, rel_l2, seeded_sd
from oracle import clip_loss_oracle as CO
from oracle import loss_oracle as LO
from oracle import lpips_oracle as LP
from oracle import seeded
from oracle import tae_oracle as TO
from test_gpu_kernel_bounds import BITS, SENTINEL, Guarded, check_stores
from test_gpu_tae import SMALL, make_tvae, tf32_off

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _affine():
    """(shift, inv_scale) of the LPIPS ScalingLayer on the device."""
    return LP.SHIFT.to(DEV), (1.0 / LP.SCALE).to(DEV)


def _sel(kind, B, T):
    if kind == "all":
        return None
    g = torch.Generator().manual_seed(B * 100 + T)
    k = max(1, T // 2)
    return torch.stack([torch.randperm(T, generator=g)[:k] for _ in range(B)])


def _L():
    import native

    return native.load()


def _ok(rc, what):
    import native

    native.check(rc, what)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _framed(Nimg, H, W, fill_interior):
    """A Guarded bf16 buffer laid out like ops.alloc_framed: [Nimg][H+2][W+2][8] + 64 slack, border and slack zero,
    interior `fill_interior` (sentinel or a value), guards sentinel."""
    n = Nimg * (H + 2) * (W + 2) * 8
    G = Guarded(n + 64, torch.bfloat16)
    G.body.zero_()
    inner = G.body[:n].view(Nimg, H + 2, W + 2, 8)[:, 1:-1, 1:-1]
    if fill_interior is None:
        inner.view(BITS[torch.bfloat16]).fill_(SENTINEL[torch.bfloat16])
    else:
        inner.copy_(fill_interior)
    return G, n


# ------------------------------------------------------------------------------------------------ kernel bounds
CASES = [(dt, T, sel, framed) for dt in ("fp32", "bf16") for T in (1, 3, 16) for sel in ("all", "partial")
         for framed in (True, False)]


@pytest.mark.parametrize("dt,T,sel,framed", CASES, ids=[f"{a}-T{b}-{c}-{'framed' if d else 'plain'}"
                                                        for a, b, c, d in CASES])
def test_clip_to_frames_equals_the_2d_kernel_on_folded_frames(dt, T, sel, framed):
    B, C, H, W = 2, 3, 37, 53
    dtype = torch.float32 if dt == "fp32" else torch.bfloat16
    gen = torch.Generator(device=DEV).manual_seed(T)
    clip = (torch.rand(B, C, T, H, W, device=DEV, generator=gen) * 2 - 1).to(dtype)
    frames = _sel(sel, B, T)
    k = T if frames is None else frames.shape[1]
    X = Guarded(clip.numel(), dtype, poison="nan")
    X.body.copy_(clip.reshape(-1))
    folded = CO.fold_frames(clip, frames).contiguous()
    fr = None if frames is None else frames.to(torch.int32).reshape(-1).to(DEV)
    fptr = 0 if fr is None else fr.data_ptr()
    L = _L()
    SHIFT, INV = _affine()
    bf = "_bf16" if dt == "bf16" else ""
    if framed:
        got, n = _framed(B * k, H, W, None)
        ref, _ = _framed(B * k, H, W, None)
        _ok(getattr(L, f"vqb_ncthw_frames_to_nhwc_pad{bf}")(X.ptr(), got.ptr(), B, C, T, H, W, 8, 1, fptr, k,
                                                             SHIFT.data_ptr(), INV.data_ptr(), _stream()), "clip fwd")
        _ok(getattr(L, f"vqb_nchw_to_nhwc_pad{bf}")(folded.data_ptr(), ref.ptr(), B * k, C, H, W, 8, 1,
                                                     SHIFT.data_ptr(), INV.data_ptr(), _stream()), "2-D fwd")
        torch.cuda.synchronize()
        assert torch.equal(got.bits(), ref.bits()), "framed buffer differs from the 2-D kernel on the folded frames"
        body = got.body[:n].view(B * k, H + 2, W + 2, 8)
        inner = body[:, 1:-1, 1:-1].contiguous().view(BITS[torch.bfloat16])
        assert not bool((inner == SENTINEL[torch.bfloat16]).any()), "an interior element was not written"
        border = body.clone()
        border[:, 1:-1, 1:-1] = 0
        assert not bool(border.view(BITS[torch.bfloat16]).any()), "the zero frame was written"
        assert not bool(got.body[n:].view(BITS[torch.bfloat16]).any()), "the 64-element slack was written"
    else:
        n = B * k * H * W * 8
        got, ref = Guarded(n, torch.bfloat16), Guarded(n, torch.bfloat16)
        _ok(getattr(L, f"vqb_ncthw_frames_to_nhwc{bf}")(X.ptr(), got.ptr(), B, C, T, H, W, 8, fptr, k,
                                                         SHIFT.data_ptr(), INV.data_ptr(), _stream()), "clip fwd")
        _ok(getattr(L, f"vqb_nchw_to_nhwc{bf}")(folded.data_ptr(), ref.ptr(), B * k, C, H, W, 8, SHIFT.data_ptr(),
                                                 INV.data_ptr(), _stream()), "2-D fwd")
        torch.cuda.synchronize()
        check_stores(got, torch.arange(n, device=DEV), "clip fwd")
        assert torch.equal(got.bits(), ref.bits()), "plain buffer differs from the 2-D kernel on the folded frames"


BWD_CASES = [(T, sel, framed) for T in (1, 3, 16) for sel in ("all", "partial") for framed in (True, False)]


@pytest.mark.parametrize("T,sel,framed", BWD_CASES, ids=[f"T{a}-{b}-{'framed' if c else 'plain'}"
                                                         for a, b, c in BWD_CASES])
def test_frames_to_clip_equals_the_2d_backward_scattered(T, sel, framed):
    B, C, H, W = 2, 3, 37, 53
    frames = _sel(sel, B, T)
    k = T if frames is None else frames.shape[1]
    gen = torch.Generator(device=DEV).manual_seed(100 + T)
    g = torch.randn(B * k, H, W, 8, device=DEV, generator=gen).bfloat16()
    g[..., C:] = float("nan")  # pad channels are never read
    if framed:
        Gin, n = _framed(B * k, H, W, g)
        body = Gin.body[:n].view(B * k, H + 2, W + 2, 8)
        body[:, 0] = body[:, -1] = float("nan")  # the frame and the slack are never read either
        body[:, :, 0] = body[:, :, -1] = float("nan")
        Gin.body[n:] = float("nan")
        gin_ptr = Gin.ptr()
        gin_bits = Gin.bits()
    else:
        Gin = Guarded(g.numel(), torch.bfloat16, poison="nan")
        Gin.body.copy_(g.reshape(-1))
        gin_ptr = Gin.ptr()
        gin_bits = Gin.bits()
    fr = None if frames is None else frames.to(torch.int32).reshape(-1).to(DEV)
    fptr = 0 if fr is None else fr.data_ptr()
    L = _L()
    _, INV = _affine()
    out = Guarded(B * C * T * H * W, torch.float32)
    img = torch.empty(B * k, C, H, W, device=DEV)
    if framed:
        _ok(L.vqb_nhwc_pad_frames_to_ncthw(gin_ptr, out.ptr(), B, C, T, H, W, 8, 1, fptr, k, INV.data_ptr(),
                                           _stream()), "clip bwd")
        _ok(L.vqb_nhwc_to_nchw_pad(gin_ptr, img.data_ptr(), B * k, C, H, W, 8, 1, INV.data_ptr(), _stream()),
            "2-D bwd")
    else:
        _ok(L.vqb_nhwc_frames_to_ncthw(gin_ptr, out.ptr(), B, C, T, H, W, 8, fptr, k, INV.data_ptr(), _stream()),
            "clip bwd")
        _ok(L.vqb_nhwc_to_nchw(gin_ptr, img.data_ptr(), B * k, C, H, W, 8, INV.data_ptr(), _stream()), "2-D bwd")
    torch.cuda.synchronize()
    check_stores(out, torch.arange(out.n, device=DEV), "clip bwd")
    ref = torch.zeros(B, T, C, H, W, device=DEV)
    idx = torch.arange(T).expand(B, T) if frames is None else frames
    for b in range(B):
        ref[b, idx[b].to(DEV)] = img[b * k:(b + 1) * k]
    got = out.body.view(B, C, T, H, W)
    assert torch.equal(got.view(torch.int32), ref.transpose(1, 2).contiguous().view(torch.int32))
    if frames is not None:
        unsel = torch.ones(B, T, dtype=torch.bool)
        for b in range(B):
            unsel[b, frames[b]] = False
        assert not bool(got.transpose(1, 2)[unsel.to(DEV)].view(torch.int32).any()), "unselected frames not +0"
    assert torch.equal(Gin.bits(), gin_bits), "the gradient input was written"


# ------------------------------------------------------------------------------------------------ modules
def _lpips():
    import utils

    m = utils.LPIPS().eval()
    m.load_state_dict(seeded_sd(LP.lpips_state_dict_shapes(), "lpips"), strict=True)
    return m.cuda()


def _patchd():
    import utils

    m = utils.PatchDiscriminator()
    m.load_state_dict(seeded_sd(LP.patchd_state_dict_shapes(), "patchd"), strict=True)
    return m.cuda()


def _clip_pair(T=3, H=32, W=48):
    x = seeded.tensor("clip_gpu/x", (2, 3, T, H, W), 1.0, "uniform").cuda()
    y = seeded.tensor("clip_gpu/y", (2, 3, T, H, W), 1.0, "uniform").cuda()
    return x, y


def _unfold(gf, frames, shape):
    B, C, T, H, W = shape
    out = torch.zeros(B, T, C, H, W, device=DEV)
    k = gf.shape[0] // B
    idx = torch.arange(T).expand(B, T) if frames is None else torch.as_tensor(frames)
    for b in range(B):
        out[b, idx[b].to(DEV)] = gf[b * k:(b + 1) * k]
    return out.transpose(1, 2)


@pytest.mark.parametrize("frames", [None, [[2, 0], [1, 2]]], ids=["all", "partial"])
@pytest.mark.parametrize("train", [False, True], ids=["eval", "train-dropout"])
def test_lpips_on_a_clip_equals_lpips_on_the_folded_frames(frames, train):
    lp = _lpips().train(train)
    lp.dropout_seeds = [11, 12, 13, 14, 15]
    x, y = _clip_pair()
    xc = x.clone().requires_grad_(True)
    vc = lp(xc, y, frames=frames)
    xf = CO.fold_frames(x, frames).contiguous().requires_grad_(True)
    vf = lp(xf, CO.fold_frames(y, frames).contiguous())
    k = 3 if frames is None else 2
    assert vc.shape == vf.shape == (2 * k, 1, 1, 1)
    torch.testing.assert_close(vc, vf, rtol=1e-5, atol=0)  # fp32 atomic order of the per-layer spatial means
    vc.mean().backward()
    vf.mean().backward()
    assert torch.equal(xc.grad, _unfold(xf.grad, frames, x.shape)), "clip gradient != folded gradient, permuted back"
    if frames is not None:
        assert not bool(xc.grad[0, :, 1].any()) and not bool(xc.grad[1, :, 0].any())


@pytest.mark.parametrize("frames", [None, [[2, 0], [1, 2]]], ids=["all", "partial"])
def test_patchd_on_a_clip_equals_patchd_on_the_folded_frames(frames):
    pd = _patchd()
    x, _ = _clip_pair()
    xc = x.clone().requires_grad_(True)
    lc = pd(xc, frames=frames)
    xf = CO.fold_frames(x, frames).contiguous().requires_grad_(True)
    lf = pd(xf)
    assert lc.shape == lf.shape == ((6 if frames is None else 4), 6)
    assert torch.equal(lc, lf)
    gy = seeded.tensor("clip_gpu/gy", tuple(lc.shape)).cuda()
    (lc * gy).sum().backward()
    (lf * gy).sum().backward()
    assert torch.equal(xc.grad, _unfold(xf.grad, frames, x.shape))


def test_bf16_clip_under_no_grad():
    lp, pd = _lpips(), _patchd()
    x, y = _clip_pair()
    xb, yb = x.bfloat16(), y.bfloat16()
    frames = [[1], [2]]
    with torch.no_grad():
        vc = lp(xb, yb, frames=frames)
        vf = lp(CO.fold_frames(xb, frames).contiguous(), CO.fold_frames(yb, frames).contiguous())
        lc = pd(xb, frames=frames)
        lf = pd(CO.fold_frames(xb, frames).contiguous())
    torch.testing.assert_close(vc, vf, rtol=1e-5, atol=0)
    assert torch.equal(lc, lf) and bool(torch.isfinite(lc).all())


# ------------------------------------------------------------------------------------------------ the training step
LR_VAE, LR_DISC = 1e-4, 1e-4


def _weights():
    m, tsd = make_tvae(SMALL, "tae_small", torch.float32)
    lsd = seeded_sd(LP.lpips_state_dict_shapes(), "lpips")
    psd = seeded_sd(LP.patchd_state_dict_shapes(), "patchd")
    return tsd, lsd, psd


def _trainer(tsd, lsd, psd, perceptual_frames=None, recompute=False, gan=True):
    import tae
    import tae_trainer
    import utils

    m = tae.TVAE(**SMALL.kwargs())
    m.load_state_dict(tsd)
    lp = utils.LPIPS().eval()
    lp.load_state_dict(lsd, strict=True)
    pd = None
    if gan:
        pd = utils.PatchDiscriminator()
        pd.load_state_dict(psd, strict=True)
        pd = pd.cuda()
    return tae_trainer.VideoTrainer(m.cuda(), lp.cuda(), pd, disc_type="hinge", use_lecam=True,
                                    perceptual_frames=perceptual_frames, lr_vae=LR_VAE, lr_disc=LR_DISC,
                                    recompute=recompute)


class OracleTrainer:
    """The same step in the oracle's autograd: fp32 (TF32 off) or under bf16 autocast (the peer); torch.optim.AdamW."""

    def __init__(self, tsd, lsd, psd, autocast, gan=True):
        self.tp = {k: v.cuda().clone().requires_grad_(True) for k, v in tsd.items()}
        self.lsd = {k: v.cuda() for k, v in lsd.items()}
        self.dp = {k: v.cuda().clone().requires_grad_("scaling_layer" not in k) for k, v in psd.items()}
        kw = dict(weight_decay=1e-3, betas=(0.9, 0.95))
        self.opt_g = torch.optim.AdamW(self.tp.values(), lr=LR_VAE, **kw)
        self.opt_d = torch.optim.AdamW([v for k, v in self.dp.items() if v.requires_grad], lr=LR_DISC, **kw)
        self.anchors = [0.0, 0.0]
        self.autocast, self.gan = autocast, gan

    def step(self, x, eps, sel):
        ac = lambda: torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.autocast)  # noqa: E731
        with ac():
            decz, z = TO.forward(self.tp, x, eps, SMALL)
        decz, z = decz.float(), z.float()
        if not self.gan:
            with ac():
                percep = CO.lpips_clip(self.lsd, LO.gradnorm(decz), x, sel).float().mean()
            vl, _ = LO.vae_loss_function(x, decz, z)
            loss = percep + vl
            self.opt_g.zero_grad()
            loss.backward()
            self.opt_g.step()
            return loss.item(), None, None
        with ac():
            real = CO.patchd_clip(self.dp, x, sel).float()
            fake = CO.patchd_clip(self.dp, decz.detach(), sel).float()
        d_loss, ar, af, _ = LO.gan_disc_loss(real, fake, "hinge")
        self.anchors = [0.9 * self.anchors[0] + 0.1 * ar, 0.9 * self.anchors[1] + 0.1 * af]
        total = d_loss + 0.1 * LO.lecam_loss(real, fake, self.anchors[0], self.anchors[1])
        self.opt_d.zero_grad()
        total.backward()
        dgrads = {k: v.grad.float().clone() for k, v in self.dp.items() if v.requires_grad}
        self.opt_d.step()
        frozen = {k: v.detach() for k, v in self.dp.items()}
        with ac():
            percep = CO.lpips_clip(self.lsd, LO.gradnorm(decz), x, sel).float().mean()
            g_fake = CO.patchd_clip(frozen, LO.gradnorm(decz, 1.0), sel).float()
        vl, _ = LO.vae_loss_function(x, decz, z)
        loss = percep - g_fake.mean() + vl
        self.opt_g.zero_grad()
        loss.backward()
        tgrads = {k: v.grad.float().clone() for k, v in self.tp.items()}
        self.opt_g.step()
        return loss.item(), tgrads, dgrads


def _eps(seed, z):
    torch.manual_seed(seed)
    return torch.randn_like(z.chunk(2, dim=1)[0])  # the draw TVAE.forward made after torch.manual_seed(seed)


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


def test_one_step_gradients_match_oracle_autograd():
    tsd, lsd, psd = _weights()
    tr = _trainer(tsd, lsd, psd, perceptual_frames=3)
    x = seeded.tensor("clip_gpu/train_x", (1, 3, 4, 32, 32), 1.0, "uniform").bfloat16().float().cuda()
    torch.manual_seed(3)
    out = tr.step(x)
    sel = tr.last_frames
    assert sel.shape == (1, 3)
    eps = _eps(3, out["z"])
    ours_t = {k: p.grad for k, p in tr.vae.named_parameters()}
    ours_d = {k: p.grad for k, p in tr.disc.named_parameters()}
    with tf32_off():
        tl, tt, td = OracleTrainer(tsd, lsd, psd, False).step(x, eps, sel)
    pl, pt, pdg = OracleTrainer(tsd, lsd, psd, True).step(x, eps, sel)
    ol = out["overall_vae_loss"].item()
    el, ep = abs(ol - tl) / abs(tl), abs(pl - tl) / abs(tl)
    print(f"\nloss ours {ol:.6f} fp32 oracle {tl:.6f} peer {pl:.6f}: rel {el:.3e} (peer {ep:.3e})")
    assert el <= 1.5 * ep + 2e-3
    assert set(ours_t) == set(tt) and set(ours_d) == set(td)
    _cos_check("TVAE parameter gradients", ours_t, tt, pt)
    _cos_check("PatchD parameter gradients", ours_d, td, pdg)


def test_ten_steps_track_the_oracle_loss_curve():
    """LPIPS + z loss (the GAN terms are held by the one-step test: the generator's hinge loss takes both signs, which
    leaves a relative deviation of the curve without a scale)."""
    tsd, lsd, psd = _weights()
    tr = _trainer(tsd, lsd, psd, perceptual_frames=2, gan=False)
    x = seeded.tensor("clip_gpu/train_x", (1, 3, 4, 32, 32), 1.0, "uniform").bfloat16().float().cuda()
    ours, sels, epss = [], [], []
    for i in range(10):
        torch.manual_seed(100 + i)
        out = tr.step(x)
        ours.append(out["overall_vae_loss"].item())
        sels.append(tr.last_frames)
        epss.append(_eps(100 + i, out["z"]))

    def curve(autocast):
        o = OracleTrainer(tsd, lsd, psd, autocast, gan=False)
        return np.array([o.step(x, e, s)[0] for e, s in zip(epss, sels)])

    with tf32_off():
        truth = curve(False)
    peer = curve(True)
    ours = np.array(ours)
    print("\nloss curve ours  ", " ".join(f"{v:.5f}" for v in ours))
    print("loss curve fp32  ", " ".join(f"{v:.5f}" for v in truth))
    print("loss curve peer  ", " ".join(f"{v:.5f}" for v in peer))
    e, pe = np.abs(ours - truth) / np.abs(truth), np.abs(peer - truth) / np.abs(truth)
    print(f"max rel deviation from the fp32 curve: ours {e.max():.3e}  bf16 autocast peer {pe.max():.3e}")
    assert e[0] < 1e-2 and e.max() <= 1.5 * pe.max() + 2e-2
    assert ours[-1] < ours[0]


def test_recompute_gives_the_plain_gradients():
    tsd, lsd, psd = _weights()
    x = seeded.tensor("clip_gpu/train_x", (1, 3, 4, 32, 32), 1.0, "uniform").bfloat16().float().cuda()

    def grads(recompute):
        tr = _trainer(tsd, lsd, psd, perceptual_frames=2, recompute=recompute)
        torch.manual_seed(7)
        tr.step(x)
        return {k: p.grad.clone() for k, p in tr.vae.named_parameters()}

    a, b, r = grads(False), grads(False), grads(True)
    ref = {k: a[k].norm().item() for k in a}
    keys = [k for k in sorted(a) if ref[k] > 1e-3 * max(ref.values())]  # not the mathematically-zero ones
    cat = lambda g: torch.cat([g[k].flatten() for k in keys])  # noqa: E731
    noise, err = rel_l2(cat(b), cat(a)), rel_l2(cat(r), cat(a))
    worst_noise = max(rel_l2(b[k], a[k]) for k in keys)
    worst = max(rel_l2(r[k], a[k]) for k in keys)
    print(f"\nrecompute vs plain over {len(keys)} tensors: rel {err:.3e}, worst tensor {worst:.3e}; plain run to "
          f"run: rel {noise:.3e}, worst tensor {worst_noise:.3e}")
    assert err <= 2 * noise + 1e-6 and worst <= 2 * worst_noise + 1e-6
