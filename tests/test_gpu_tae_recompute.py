"""GPU (-m gpu): ResnetBlock recompute of the video autoencoder (tae.enable_training(..., recompute=True)).

The recompute path must compute what the plain training path computes. The forward is bit-identical, and so are the
activations the backward rebuilds (checked against the tensors the plain path saves). The backward then runs the same
kernels, so a recompute gradient may differ from a plain run only as much as plain runs differ from each other (the
GroupNorm backward's and column sums' fp32 atomics). That noise is heavy-tailed: measured on an H100, one plain pair's
relative L2 difference on a bias gradient ranged over 5x, and a column sum outside every ResnetBlock (decoder.conv_out's
bias) agreed bit for bit in three plain runs and differed in its last bits in the fourth. So the spread is taken from
three plain runs, and per tensor the relative L2 difference from plain run 1 is at most 10x the largest plain-plain
difference + 1e-6 (1e-6 alone where the plain runs agree bit for bit; worst ratio seen 5.8). Over all tensors the
median of that ratio is at most 1.5: a systematic difference moves the median, noise does not (0.86 to 1.16 measured).
The recompute gradients are also held to the oracle bounds of test_gpu_tae_train.py.
"""
import itertools

import numpy as np
import pytest
import torch

from helpers import cosine, rel_l2
from oracle import seeded
from oracle import tae_oracle as TO
from test_gpu_tae import SMALL, make_tvae, tf32_off
from test_gpu_tae_train import FLOOR, _loss, _oracle_step, check

pytestmark = pytest.mark.gpu

H64 = TO.TAEConfig(ch=64, ch_mult=(1, 2, 8), num_res_blocks=1, z_channels=4, resolution=32)
CONFIGS = {
    "tae_small": (SMALL, "tae_small", (1, 3, 4, 16, 24), 32),
    "heads64_two_levels": (H64, "tae_h64t", (1, 3, 8, 32, 48), 64),
}


def _resnet_blocks(m):
    import tae

    return [s for s in m.modules() if isinstance(s, tae.ResnetBlock)]


def _step(m, x, recompute, seed=3):
    """One seeded forward + backward -> (decz, z, loss, {name: grad}, grad of x)."""
    import tae

    tae.enable_training(m, recompute=recompute)
    m.zero_grad(set_to_none=True)
    xi = x.clone().requires_grad_(True)
    torch.manual_seed(seed)
    decz, z = m(xi)
    loss = _loss(decz, xi, z)
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    return decz.detach(), z.detach(), loss.detach(), grads, xi.grad


def _same_as_plain(what, rec, plains):
    """-> None where the plain runs agree bit for bit, else rel_l2(rec, plain 1) / plain spread."""
    spread = max(rel_l2(a, b) for a, b in itertools.combinations(plains, 2))
    d = rel_l2(rec, plains[0])
    assert d <= 10 * spread + 1e-6, (what, d, spread)
    return d / spread if spread > 0 else None


def _check_grads_same(what, rec, plains):
    assert all(set(rec) == set(p) for p in plains), what
    ratios = {}
    for k in sorted(rec):
        r = _same_as_plain(f"{what} {k}", rec[k], [p[k] for p in plains])
        if r is not None:
            ratios[k] = r
    worst = max(ratios, key=ratios.get) if ratios else None
    med = float(np.median(list(ratios.values()))) if ratios else 0.0
    print(f"\n{what}: {len(rec) - len(ratios)}/{len(rec)} tensors bit-identical across the plain runs; "
          f"others: median ratio to the plain spread {med:.2f}, worst {ratios.get(worst, 0.0):.2f} ({worst})")
    assert med <= 1.5, (what, med)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("C", [64, 256, 1024])
def test_gn_silu_apply_reproduces_the_forward_bit_for_bit(C, silu):
    """vqb_gn_silu_apply with the mr that vqb_gn_silu_fwd produced gives that call's y bit for bit, and writes exactly
    the addressed elements: a NaN-sentinel output with 4 KB guard bands on both sides."""
    import native
    import ops

    g = torch.Generator(device="cuda").manual_seed(C + silu)
    N, HW = 2, 1037  # ragged: not a multiple of any chunk or row count
    x = (torch.randn(N, 17, 61, C, device="cuda", generator=g) * 3 + 0.5).bfloat16()
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    y_ref, mr = ops.gn_silu_fwd(x, gamma, beta, 32, 1e-6, bool(silu))
    guard = 2048  # bf16 elements = 4 KB
    n = N * HW * C
    buf = torch.full((guard + n + guard,), float("nan"), device="cuda", dtype=torch.bfloat16)
    sentinel = buf[:1].view(torch.int16).clone()
    y = buf[guard:guard + n]
    L = native.load()
    native.check(L.vqb_gn_silu_apply(x.data_ptr(), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(), mr.data_ptr(), N,
                                     HW, C, 32, silu, native.stream_ptr()), "gn_silu_apply")
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), y_ref.reshape(-1).view(torch.int16))
    assert bool((buf[:guard].view(torch.int16) == sentinel).all())
    assert bool((buf[guard + n:].view(torch.int16) == sentinel).all())
    assert torch.equal(ops.gn_silu_apply(x, gamma, beta, mr, bool(silu)).view(torch.int16), y_ref.view(torch.int16))


# ------------------------------------------------------------------------------------------------ module
@pytest.mark.parametrize("name", list(CONFIGS))
def test_recompute_forward_and_gradients_match_the_plain_path(name):
    cfg, tag, shape, head_dim = CONFIGS[name]
    m, sd = make_tvae(cfg, tag, torch.float32)
    m.train()
    assert m.encoder.mid.attn_1.head_dim == head_dim
    x = seeded.tensor(f"{tag}/x", shape, 1.0, "uniform").bfloat16().float().cuda()
    plains = [_step(m, x, False) for _ in range(3)]
    rc = _step(m, x, True)
    for i, what in enumerate(("decz", "z", "loss")):
        assert torch.equal(rc[i], plains[0][i]), f"{name}: recompute {what} differs from the plain training forward"
    _check_grads_same(name, rc[3], [p[3] for p in plains])
    _same_as_plain(f"{name} input grad", rc[4], [p[4] for p in plains])

    # the oracle bounds of test_gpu_tae_train.py, on the recompute gradients
    torch.manual_seed(3)
    eps = torch.randn_like(rc[1].chunk(2, dim=1)[0])
    with tf32_off():
        tl, tg, tx = _oracle_step(cfg, sd, x.cpu(), eps, torch.float32)
    pl, pg, px = _oracle_step(cfg, sd, x.cpu(), eps, torch.bfloat16)
    el, ep = abs(rc[2].item() - tl.item()) / abs(tl.item()), abs(pl.item() - tl.item()) / abs(tl.item())
    assert el <= 1.5 * ep + FLOOR
    check(f"{name} recompute input grad", rc[4], tx, px)
    keys = sorted(tg)
    grads = rc[3]
    ref = np.array([tg[k].norm().item() for k in keys])
    big = ref > 1e-3 * ref.max()
    ours_n = np.array([grads[k].norm().item() for k in keys])[big] / ref[big]
    peer_n = np.array([pg[k].norm().item() for k in keys])[big] / ref[big]
    cos = np.array([cosine(grads[k], tg[k]) for k in keys])[big]
    pcos = np.array([cosine(pg[k], tg[k]) for k in keys])[big]
    print(f"  recompute, {big.sum()} tensors: cosine min {cos.min():.5f} (peer {pcos.min():.5f}); norm ratio "
          f"[{ours_n.min():.4f}, {ours_n.max():.4f}] (peer [{peer_n.min():.4f}, {peer_n.max():.4f}])")
    bad = [(k, round(c, 5), round(pc, 5)) for k, c, pc in zip(np.array(keys)[big], cos, pcos)
           if 1 - c > 1.5 * (1 - pc) + 5e-3]
    assert not bad, bad
    assert np.abs(ours_n - 1).max() <= 1.5 * np.abs(peer_n - 1).max() + 0.02


# ------------------------------------------------------------------------------------------------ memory, launches
def _saved(fn):
    """-> list of the tensors autograd saves while fn() runs."""
    saved = []

    def pack(t):
        saved.append(t)
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        out = fn()
    return saved, out


@pytest.mark.parametrize("cin,cout", [(64, 128), (128, 128)])
def test_saved_tensors_per_block_drop_to_the_input(cin, cout):
    """Counted from the shapes: without recompute a ResnetBlock keeps x, hn, h and h2 (bf16) and two [N, 32, 2] fp32
    GroupNorm records; with recompute, x and the two records. The parameters it saves are its own."""
    import tae

    torch.manual_seed(0)
    blk = tae.ResnetBlock(cin, cout).cuda()
    N, T, H, W = 2, 4, 8, 12
    x = torch.randn(N, cin, T, H, W, device="cuda", requires_grad=True)
    params = {p.data_ptr(): p for p in blk.parameters()}
    vox = N * T * H * W
    stats = 2 * N * 32 * 2 * 4
    want = {False: 2 * vox * (2 * cin + 2 * cout) + stats, True: 2 * vox * cin + stats}
    for recompute in (False, True):
        tae.enable_training(blk, recompute=recompute)
        saved, out = _saved(lambda: blk(x))
        acts = {t.data_ptr(): t.numel() * t.element_size() for t in saved if t.data_ptr() not in params}
        pp = {t.data_ptr() for t in saved if t.data_ptr() in params}
        print(f"\nResnetBlock({cin}, {cout}) recompute={recompute}: {sum(acts.values())} saved activation bytes "
              f"in {len(acts)} tensors, {len(pp)} parameters")
        assert sum(acts.values()) == want[recompute], (recompute, sorted(acts.values()))
        assert len(acts) == (3 if recompute else 6)
        if recompute:
            assert pp == set(params)
        out.sum().backward()


@pytest.mark.parametrize("cin,cout", [(256, 32), (128, 128)])
def test_rebuilt_activations_equal_the_plain_saved_tensors(cin, cout):
    """What the recompute backward rebuilds from the saved x and mr records (GroupNorm apply, conv1, GroupNorm apply)
    is, bit for bit, the hn, h and h2 the plain training path saves."""
    import ops
    import tae

    torch.manual_seed(0)
    blk = tae.ResnetBlock(cin, cout).cuda()
    x = torch.randn(1, cin, 4, 16, 24, device="cuda", requires_grad=True)
    params = {p.data_ptr() for p in blk.parameters()}
    tae.enable_training(blk)
    plain = [t for t in _saved(lambda: blk(x))[0] if t.data_ptr() not in params]
    tae.enable_training(blk, recompute=True)
    xs, mr1, mr2 = [t for t in _saved(lambda: blk(x))[0] if t.data_ptr() not in params]
    N, T, H, W, C = xs.shape
    with torch.no_grad():
        hn = ops.gn_silu_apply(xs.view(N, T * H, W, C), blk.norm1.weight, blk.norm1.bias, mr1, True)
        h = ops.conv3d(hn.view(N, T, H, W, C), blk.conv1.weight, blk.conv1.bias, blk.conv1._packed, "s1")
        h2 = ops.gn_silu_apply(h.view(N, T * H, W, -1), blk.norm2.weight, blk.norm2.bias, mr2, True)
    # saved by the plain path in this order: x (norm1), mr1, hn (conv1), h (norm2), mr2, [x (nin_shortcut)], h2 (conv2)
    for what, a, b in (("x", plain[0], xs), ("mr1", plain[1], mr1), ("hn", plain[2], hn), ("h", plain[3], h),
                       ("mr2", plain[4], mr2), ("h2", plain[-1], h2)):
        assert torch.equal(a.reshape(-1), b.reshape(-1)), what


# peak allocated memory of a forward + backward at 16x256^2, ch=64, batch 1 (tools/tae_train_bench.py's smaller clip):
# with recompute over without. Measured on an H100 80GB HBM3: 1.97 GiB against 4.24 GiB, a ratio of 0.465.
MEMORY_RATIO_BOUND = 0.55


def test_recompute_lowers_peak_memory():
    import tae

    cfg = TO.TAEConfig(ch=64)
    torch.manual_seed(1)
    m = tae.TVAE(**cfg.kwargs()).cuda()
    torch.manual_seed(0)
    x = torch.rand(1, 3, 16, 256, 256, device="cuda") * 2 - 1

    def peak(recompute):
        tae.enable_training(m, recompute=recompute)
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        decz, z = m(x)
        _loss(decz, x, z).backward()
        del decz, z
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    peak(False)  # packs the weights, plans the shapes
    plain, rec = peak(False), peak(True)
    print(f"\npeak allocated, forward + backward at 16x256^2 ch=64: plain {plain / 2 ** 30:.2f} GiB, recompute "
          f"{rec / 2 ** 30:.2f} GiB, ratio {rec / plain:.3f}")
    assert rec <= MEMORY_RATIO_BOUND * plain


def test_recompute_adds_exactly_conv1_and_two_groupnorm_applies_per_block():
    """native.launch_count() of a recompute step minus a plain step = (one conv1 launch + two GroupNorm apply launches)
    per ResnetBlock: no extra column sum or statistics pass."""
    import native

    m, _ = make_tvae(H64, "tae_h64t", torch.float32)
    x = seeded.tensor("tae_h64t/x", (1, 3, 8, 32, 48), 1.0, "uniform").cuda()
    for rc in (False, True):  # warm-up: packs every forward and transposed operand
        _step(m, x, rc)

    def count(recompute):
        torch.cuda.synchronize()
        n0 = native.launch_count()
        _step(m, x, recompute)
        return native.launch_count() - n0

    plain, rec = count(False), count(True)
    nblocks = len(_resnet_blocks(m))
    print(f"\nlaunches per step: plain {plain}, recompute {rec}, {nblocks} ResnetBlocks")
    assert rec - plain == nblocks * (1 + 2)


# ------------------------------------------------------------------------------------------------ training
def test_adamw_steps_follow_the_plain_curve_and_repack_the_weights():
    import ops
    import tae

    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").bfloat16().float().cuda()
    eps = seeded.tensor("tae_small/eps_train", (1, 4, 2, 8, 12), 1.0).cuda()

    def curve(recompute):
        m, _ = make_tvae(SMALL, "tae_small", torch.float32)
        tae.enable_training(m.train(), recompute=recompute)
        opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
        out = []
        for _ in range(10):
            opt.zero_grad()
            z = m.encoder(x)
            loss = _loss(m.decoder(ops.gauss_reparam_train(z, eps)), x, z)
            loss.backward()
            opt.step()
            out.append(loss.item())
        return m, torch.tensor(out, dtype=torch.float64)

    plains = [curve(False)[1] for _ in range(3)]
    m, cr = curve(True)
    print("\nloss curve plain    ", " ".join(f"{v:.7f}" for v in plains[0].tolist()))
    print("loss curve recompute", " ".join(f"{v:.7f}" for v in cr.tolist()))
    _same_as_plain("loss curve", cr, plains)
    fresh = tae.TVAE(**SMALL.kwargs())
    fresh.load_state_dict({k: v.detach().cpu() for k, v in m.state_dict().items()})
    fresh = fresh.cuda().eval()
    with torch.no_grad():
        assert torch.equal(m.encoder(x), fresh.encoder(x))
        assert torch.equal(m.decoder(eps), fresh.decoder(eps))


# ------------------------------------------------------------------------------------------------ composition
def test_frozen_parameters_give_the_plain_input_gradient():
    m, _ = make_tvae(SMALL, "tae_small", torch.float32)
    m.requires_grad_(False)
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").cuda()
    plains = [_step(m, x, False) for _ in range(3)]
    rc = _step(m, x, True)
    assert not rc[3] and rc[4] is not None and rc[4].abs().sum() > 0
    _same_as_plain("frozen input grad", rc[4], [p[4] for p in plains])


def test_decoder_only_opt_in():
    import tae

    m, _ = make_tvae(SMALL, "tae_small", torch.float32)
    m.encoder.requires_grad_(False)
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").cuda()

    def run(recompute):
        tae.enable_training(m, False)
        tae.enable_training(m.decoder, recompute=recompute)
        m.zero_grad(set_to_none=True)
        torch.manual_seed(3)
        saved, (decz, z) = _saved(lambda: m(x))
        _loss(decz, x, z).backward()
        return sum(t.numel() * t.element_size() for t in saved), {k: p.grad.clone() for k, p in
                                                                   m.decoder.named_parameters()}

    plains = [run(False) for _ in range(3)]
    br, gr = run(True)
    assert all(p.grad is None for p in m.encoder.parameters())
    assert br < plains[0][0] == plains[1][0]  # the decoder's blocks saved less
    _check_grads_same("decoder-only opt-in", gr, [g for _, g in plains])


def test_weight_changed_in_place_between_forward_and_backward_raises():
    import tae

    m, _ = make_tvae(SMALL, "tae_small", torch.float32)
    tae.enable_training(m.train(), recompute=True)
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").cuda()
    decz, z = m(x)
    loss = _loss(decz, x, z)
    with torch.no_grad():
        m.decoder.up[0].block[0].conv1.weight.mul_(1.01)
    with pytest.raises(RuntimeError, match="inplace"):
        loss.backward()
