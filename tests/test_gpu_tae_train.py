"""GPU (-m gpu): training of the video autoencoder (tae.enable_training) on the native kernels.

Tolerance rule (as in test_gpu_tae.py). Truth is fp32 with TF32 off on the SAME bf16-rounded weights and inputs. The peer
is the same arithmetic with bf16 weights and inputs (cuDNN). Kernel level: rel_L2(ours) <= 1.5 x rel_L2(peer) + FLOOR
per gradient. Module level: every parameter tensor's cosine error within 1.5x the peer's for that tensor plus 5e-3,
and (as in test_gpu_parity.py) the worst gradient-norm ratio error over all tensors within 1.5x the peer's plus 2 %.
Every check prints ours next to the peer's.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import cosine, rel_l2
from oracle import seeded
from oracle import tae_oracle as TO
from test_gpu_tae import SMALL, _ncthw, _nthwc, make_tvae, tf32_off

pytestmark = pytest.mark.gpu

FLOOR = 2e-3


def check(what, ours, truth, peer):
    assert ours.shape == truth.shape == peer.shape, (what, ours.shape, truth.shape, peer.shape)
    assert bool(torch.isfinite(ours.float()).all()), what
    e, p = rel_l2(ours, truth), rel_l2(peer, truth)
    print(f"\n{what}: ours rel {e:.3e}  bf16 cuDNN peer rel {p:.3e}  (vs fp32 truth)")
    assert e <= 1.5 * p + FLOOR, (what, e, p)


def _ref(kind, x, w, b):
    if kind == "s1":
        return F.conv3d(x, w, b, padding=1)
    if kind == "s2":
        return F.conv3d(F.pad(x, (0, 1, 0, 1, 0, 1)), w, b, stride=2)
    if kind == "p1":
        return F.conv3d(x, w, b)
    return F.conv3d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, b, padding=1)


def _ref_grads(kind, x, w, b, dy):
    x, w, b = (u.detach().clone().requires_grad_(True) for u in (x, w, b))
    return torch.autograd.grad(_ref(kind, x, w, b), (x, w, b), dy.to(x.dtype))


# ------------------------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("kind", ["s1", "s2", "up", "p1"])
@pytest.mark.parametrize("Cin,Cout", [(3, 64), (64, 3), (64, 8), (256, 256)])
def test_conv3d_gradients_match_autograd(kind, Cin, Cout):
    import ops

    g = torch.Generator(device="cuda").manual_seed(Cin * 1000 + Cout)
    T, H, W = (6, 10, 22) if kind == "s2" else (5, 9, 21)  # ragged tiles; s2 needs even extents
    if Cin == 256:
        T, H, W = (4, 6, 10) if kind == "s2" else (3, 5, 9)
    ks = (1, 1, 1) if kind == "p1" else (3, 3, 3)
    x = (torch.rand(2, Cin, T, H, W, device="cuda", generator=g) - 0.5).bfloat16().float()
    w = (torch.randn(Cout, Cin, *ks, device="cuda", generator=g) * 0.2).bfloat16().float()
    b = torch.randn(Cout, device="cuda", generator=g) * 0.1
    with torch.no_grad():
        yshape = _ref(kind, x, w, b).shape
    dy = (torch.randn(*yshape, device="cuda", generator=g)).bfloat16().float()
    with tf32_off():
        tx, tw, tb = _ref_grads(kind, x, w, b, dy)
    px, pw, pb = _ref_grads(kind, x.bfloat16(), w.bfloat16(), b.bfloat16(), dy)
    wp = w.clone().requires_grad_(True)
    bp = b.clone().requires_grad_(True)
    xa = _nthwc(x).requires_grad_(True)
    cache = ops.PackedCache()
    if kind == "up":
        y = ops.upsample_conv3d_train(xa, wp, bp, cache)
    else:
        y = ops.conv3d_train(xa, wp, bp, cache, kind)
    y.backward(_nthwc(dy))
    tag = f"{kind} Cin={Cin} Cout={Cout}"
    check(f"{tag} dgrad", _ncthw(xa.grad, Cin), tx, px)
    check(f"{tag} wgrad", wp.grad, tw, pw)
    check(f"{tag} bias grad", bp.grad, tb, pb)
    if kind in ("s1", "s2"):  # module-boundary form: NCTHW fp32 output, gradient back through vqb_nchw_to_nhwc
        wq = w.clone().requires_grad_(True)
        xb = _nthwc(x).requires_grad_(True)
        yo = ops.conv3d_train(xb, wq, None, ops.PackedCache(), kind, None, True)
        assert yo.shape == yshape and yo.dtype == torch.float32
        yo.backward(dy)
        check(f"{tag} NCTHW-out dgrad", _ncthw(xb.grad, Cin), tx, px)
        check(f"{tag} NCTHW-out wgrad", wq.grad, tw, pw)


@pytest.mark.parametrize("head_dim", [32, 64])
def test_attention_backward_matches_sdpa(head_dim):
    import ops

    g = torch.Generator(device="cuda").manual_seed(head_dim + 1)
    N, T, heads = 2, 6144, 8
    C = heads * head_dim
    qkv = torch.randn(N, 6, 32, 32, 3 * C, device="cuda", generator=g).bfloat16()
    dout = torch.randn(N, 6, 32, 32, C, device="cuda", generator=g).bfloat16()
    q0 = qkv.clone().requires_grad_(True)
    ops.attention_hd_train(q0, heads, head_dim).backward(dout)

    def sdpa_grad(u, d):
        u = u.detach().clone().requires_grad_(True)
        q, k, v = (a.reshape(N, T, heads, head_dim).permute(0, 2, 1, 3) for a in u.reshape(N, T, 3 * C).chunk(3, -1))
        o = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(u.shape[:-1] + (C,))
        o.backward(d.to(u.dtype))
        return u.grad

    with tf32_off():
        truth = sdpa_grad(qkv.float(), dout)
    peer = sdpa_grad(qkv, dout)
    for i, part in enumerate("qkv"):
        sl = slice(i * C, (i + 1) * C)
        check(f"attention heads of {head_dim} d{part}", q0.grad[..., sl], truth[..., sl], peer[..., sl])


def test_gauss_reparam_backward_matches_autograd():
    import ops

    g = torch.Generator(device="cuda").manual_seed(7)
    z = torch.randn(2, 8, 3, 5, 7, device="cuda", generator=g) * 2
    z[:, 4:, 0, 0, :3] = -3.0  # logvar exactly at the clamp: the gradient passes (torch's clamp backward)
    z[:, 4:, 0, 1, :3] = -3.5  # below it: no gradient
    eps = torch.randn(2, 4, 3, 5, 7, device="cuda", generator=g)
    gout = torch.randn(2, 4, 3, 5, 7, device="cuda", generator=g)
    zo = z.clone().requires_grad_(True)
    ops.gauss_reparam_train(zo, eps).backward(gout)
    zr = z.double().requires_grad_(True)
    TO.reg(zr, eps.double()).backward(gout.double())
    assert bool((zr.grad[:, 4:, 0, 0, :3] != 0).all()) and bool((zr.grad[:, 4:, 0, 1, :3] == 0).all())
    assert bool((zo.grad[:, 4:, 0, 0, :3] != 0).all()) and bool((zo.grad[:, 4:, 0, 1, :3] == 0).all())
    err = (zo.grad.double() - zr.grad).abs()
    bound = 2.0 ** -20 * (zr.grad.abs() + gout.double().abs().repeat(1, 2, 1, 1, 1))
    print(f"\ngauss_reparam backward: max abs err {err.max().item():.3e}")
    assert bool((err <= bound).all())


# ------------------------------------------------------------------------------------------------ module level
def _loss(decz, x, z):
    return F.mse_loss(decz, x) + 0.1 * z.pow(2).mean()


def _oracle_step(cfg, sd, x, eps, dtype):
    """-> (loss, {name: grad}, grad of x) of the oracle's autograd in `dtype` on the GPU."""
    p = {k: v.cuda().to(dtype).requires_grad_(True) for k, v in sd.items()}
    xi = x.cuda().to(dtype).requires_grad_(True)
    decz, z = TO.forward(p, xi, eps.cuda().to(dtype), cfg)
    loss = _loss(decz.float(), xi.float(), z.float())
    loss.backward()
    return loss.detach(), {k: v.grad.float() for k, v in p.items()}, xi.grad.float()


def _grad_parity(what, cfg, tag, x, head_dim):
    import tae

    m, sd = make_tvae(cfg, tag, torch.float32)
    assert m.encoder.mid.attn_1.head_dim == m.decoder.mid.attn_1.head_dim == head_dim
    tae.enable_training(m.train())
    xi = x.cuda().requires_grad_(True)
    torch.manual_seed(3)
    decz, z = m(xi)
    torch.manual_seed(3)
    eps = torch.randn_like(z.chunk(2, dim=1)[0])  # the draw TVAE.forward made
    loss = _loss(decz, xi, z)
    loss.backward()
    with tf32_off():
        tl, tg, tx = _oracle_step(cfg, sd, x, eps, torch.float32)
    pl, pg, px = _oracle_step(cfg, sd, x, eps, torch.bfloat16)
    el, ep = abs(loss.item() - tl.item()) / abs(tl.item()), abs(pl.item() - tl.item()) / abs(tl.item())
    print(f"\n{what}: loss rel {el:.3e} (peer {ep:.3e})")
    assert el <= 1.5 * ep + FLOOR
    check(f"{what} input grad", xi.grad, tx, px)
    params = dict(m.named_parameters())
    keys = sorted(params)
    assert set(keys) == set(tg)
    ref = np.array([tg[k].norm().item() for k in keys])
    big = ref > 1e-3 * ref.max()  # mathematically-zero gradients (a bias in front of a GroupNorm) carry only noise
    ours_n = np.array([params[k].grad.norm().item() for k in keys])[big] / ref[big]
    peer_n = np.array([pg[k].norm().item() for k in keys])[big] / ref[big]
    cos = np.array([cosine(params[k].grad, tg[k]) for k in keys])[big]
    pcos = np.array([cosine(pg[k], tg[k]) for k in keys])[big]
    print(f"  {big.sum()} tensors: cosine min {cos.min():.5f} (peer {pcos.min():.5f}); norm ratio "
          f"[{ours_n.min():.4f}, {ours_n.max():.4f}] (peer [{peer_n.min():.4f}, {peer_n.max():.4f}])")
    # cosine per tensor against the peer's cosine for the SAME tensor: one wrong tensor (a dropped tap class, a stale
    # bias column sum) cannot hide behind the peer's worst tensor elsewhere
    bad = [(k, round(c, 5), round(pc, 5)) for k, c, pc in zip(np.array(keys)[big], cos, pcos)
           if 1 - c > 1.5 * (1 - pc) + 5e-3]
    assert not bad, bad
    assert np.abs(ours_n - 1).max() <= 1.5 * np.abs(peer_n - 1).max() + 0.02


def test_small_config_gradients_match_oracle_autograd():
    """Heads of 32, one Down/Up level."""
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").bfloat16().float()
    _grad_parity("tae_small", SMALL, "tae_small", x, head_dim=32)


def test_heads_of_64_two_level_gradients_match_oracle_autograd():
    """Attention blocks of 512 channels (8 heads of 64), two Down/Up levels."""
    cfg = TO.TAEConfig(ch=64, ch_mult=(1, 2, 8), num_res_blocks=1, z_channels=4, resolution=32)
    x = seeded.tensor("tae_h64t/x", (1, 3, 8, 32, 48), 1.0, "uniform").bfloat16().float()
    _grad_parity("heads-of-64 two levels", cfg, "tae_h64t", x, head_dim=64)


def test_frozen_parameters_give_the_input_gradient():
    import tae

    m, _ = make_tvae(SMALL, "tae_small", torch.float32)
    tae.enable_training(m.requires_grad_(False))
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").cuda().requires_grad_(True)
    decz, z = m(x)
    _loss(decz, x, z).backward()
    assert x.grad is not None and bool(torch.isfinite(x.grad).all()) and x.grad.abs().sum() > 0
    assert all(p.grad is None for p in m.parameters())


# ------------------------------------------------------------------------------------------------ training
def test_adamw_steps_track_the_oracle_and_repack_the_weights():
    """10 AdamW steps from the same bf16-rounded weights: the loss curve of ours against the fp32 oracle (TF32 off), held
    to 1.5x the deviation of the same steps under bf16 autocast (cuDNN) plus 2 %. After the steps a no-grad forward
    equals, bit for bit, a fresh module loaded with the stepped weights (the post-step hook re-packed every operand)."""
    import ops
    import tae

    m, sd = make_tvae(SMALL, "tae_small", torch.float32)
    tae.enable_training(m.train())
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").bfloat16().float().cuda()
    eps = seeded.tensor("tae_small/eps_train", (1, 4, 2, 8, 12), 1.0).cuda()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
    ours = []
    for _ in range(10):
        opt.zero_grad()
        z = m.encoder(x)
        loss = _loss(m.decoder(ops.gauss_reparam_train(z, eps)), x, z)
        loss.backward()
        opt.step()
        ours.append(loss.item())
    fresh = tae.TVAE(**SMALL.kwargs())
    fresh.load_state_dict({k: v.detach().cpu() for k, v in m.state_dict().items()})
    fresh = fresh.cuda().eval()
    with torch.no_grad():
        assert torch.equal(m.encoder(x), fresh.encoder(x))
        assert torch.equal(m.decoder(eps), fresh.decoder(eps))

    def oracle_curve(autocast):
        ref = {k: v.cuda().clone().requires_grad_(True) for k, v in sd.items()}
        ropt = torch.optim.AdamW(ref.values(), lr=1e-4)
        out = []
        for _ in range(10):
            ropt.zero_grad()
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                rd, rz = TO.forward(ref, x, eps, SMALL)
                rl = _loss(rd.float(), x, rz.float())
            rl.backward()
            ropt.step()
            out.append(rl.item())
        return np.array(out)

    with tf32_off():
        truth = oracle_curve(False)
    peer = oracle_curve(True)
    ours = np.array(ours)
    print("\nloss curve ours  ", " ".join(f"{v:.5f}" for v in ours))
    print("loss curve fp32  ", " ".join(f"{v:.5f}" for v in truth))
    print("loss curve peer  ", " ".join(f"{v:.5f}" for v in peer))
    e, pe = np.abs(ours - truth) / truth, np.abs(peer - truth) / truth
    print(f"max rel deviation from the fp32 curve: ours {e.max():.3e}  bf16 autocast peer {pe.max():.3e}")
    assert e[0] < 1e-2 and e.max() <= 1.5 * pe.max() + 2e-2
    assert ours[-1] < ours[0]


def test_opt_in_refusals_launch_nothing():
    import native
    import tae

    m, _ = make_tvae(SMALL, "tae_small", torch.float32)
    x = torch.zeros(1, 3, 4, 16, 24, device="cuda")
    n0 = native.launch_count()
    with pytest.raises(RuntimeError, match="no_grad"):
        m(x)
    b = tae.enable_training(m.bfloat16())
    with pytest.raises(RuntimeError, match="inference-only"):
        b(x.bfloat16())
    with pytest.raises(RuntimeError, match="float16"):
        b.half()(x.half())
    torch.cuda.synchronize()
    assert native.launch_count() == n0
