"""GPU (-m gpu): ResnetBlock recompute of the image autoencoder (ae.enable_recompute, Trainer(..., recompute=True)).

The recompute node runs the kernels of the plain training path. Where conv1 cannot fuse the GroupNorm statistics into
its epilogue, its forward is bit-identical to the plain one; where it does, the statistics' fp32 atomics make every
later activation vary in its last bits from run to run, on the plain path as much as on this one. The activations the
backward rebuilds are bit-identical to the forward's, because conv1 stores the same bf16 values with and without the
statistics epilogue (checked at kernel level below). The gradients then differ from a plain run only as much as plain
runs differ from each other, so they are compared like tests/test_gpu_tae_recompute.py does: per tensor the relative
L2 difference from plain run 1 is at most 10x the largest difference among three plain runs + 1e-6, and over all
tensors the median of that ratio is at most 1.5 (a systematic difference moves the median, noise does not). The
recompute gradients are also held to the oracle bounds of tests/test_gpu_parity.py.
"""
import itertools

import numpy as np
import pytest
import torch

from helpers import cosine, golden, rel_l2
from oracle import seeded
from oracle import vae_oracle as VO
from test_gpu_parity import COS_TOL, build_vae, check_grads

pytestmark = pytest.mark.gpu


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


def _blocks(m):
    import ae

    return [s for s in m.modules() if isinstance(s, ae.ResnetBlock)]


def _saved(fn):
    """-> (tensors autograd saves while fn() runs, fn())."""
    saved = []

    def pack(t):
        saved.append(t)
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        out = fn()
    return saved, out


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ kernel
# (N, H, W, Cout): BLOCK_N 16 / 64 / 128 (Cout 512: four column tiles), a ragged last column tile (192), ragged pixel
# tiles (20x24) and tiles that span images (8x8)
CONV_SHAPES = [(2, 16, 16, 16), (2, 16, 16, 64), (2, 32, 32, 128), (1, 16, 32, 512), (2, 16, 16, 192),
               (2, 20, 24, 128), (4, 8, 8, 128)]


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("N,H,W,Cout", CONV_SHAPES)
def test_conv_stores_the_same_values_with_and_without_the_statistics_epilogue(N, H, W, Cout, bias):
    """The 3x3 stride-1 conv_gemm_kernel writes the same bf16 output with VQB_EPI_STATS as without it (the recompute
    rebuilds conv1's output without the statistics). Where the epilogue cannot produce statistics (Cout not a multiple
    of 64, ragged pixel tiles, tiles across images) the kernel refuses VQB_EPI_STATS, so the forward ran without it
    too, and the rebuild is the same launch: it must then be deterministic."""
    import ops
    import plans

    Cin = 64
    g = torch.Generator(device="cuda").manual_seed(N * H * W + Cout + bias)
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).bfloat16()
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * 0.05
    b = torch.randn(Cout, device="cuda", generator=g) if bias else None
    geo = plans.geom_s1(N, H, W, Cin, 3)
    wp = ops.PackedCache().get(w, ("fwd", "s1"), geo.tapmap, False, Cin)
    ostr = plans.nhwc_strides(H, W, Cout)

    def run(stats=None):
        out = torch.full((N, H, W, Cout), float("nan"), device="cuda", dtype=torch.bfloat16)
        ops.run_conv_gemm(geo, x, wp, Cout, out, ostr, bias=b, stats=stats)
        return out

    ref = run()
    assert not torch.isnan(ref).any()
    ok = ops.conv_stats_supported(geo, Cout, ostr)
    expected_ok = Cout % 64 == 0 and (N, H, W) in ((2, 16, 16), (2, 32, 32), (1, 16, 32))
    assert ok == expected_ok, (N, H, W, Cout)
    if ok:
        st = torch.zeros(N, Cout, 2, device="cuda")
        with_stats = run(st)
        torch.cuda.synchronize()
        assert torch.equal(_bits(with_stats), _bits(ref))
        want = torch.stack([ref.float().sum((1, 2)), ref.float().pow(2).sum((1, 2))], -1)
        assert torch.allclose(st, want, rtol=1e-4, atol=1e-2)  # the epilogue did run
    else:
        with pytest.raises(RuntimeError, match="VQB_EPI_STATS unsupported"):
            run(torch.zeros(N, Cout, 2, device="cuda"))
        assert torch.equal(_bits(run()), _bits(ref))


@pytest.mark.parametrize("C", [64, 256, 512])
def test_gn_silu_apply_reproduces_the_fused_statistics_forward(C):
    """vqb_gn_silu_apply with the mr that vqb_gn_silu_fwd_pre finalised from column sums gives that call's y bit for
    bit, and writes exactly the addressed elements: a NaN-sentinel output with 4 KB guard bands on both sides."""
    import native
    import ops

    g = torch.Generator(device="cuda").manual_seed(C)
    N, H, W = 2, 16, 24
    x = (torch.randn(N, H, W, C, device="cuda", generator=g) * 2 + 0.3).bfloat16()
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    xf = x.float()
    chsums = torch.stack([xf.sum((1, 2)), xf.pow(2).sum((1, 2))], -1).contiguous()
    y_ref, mr = ops.gn_silu_fwd_pre(x, gamma, beta, chsums, 32, 1e-6, True)
    guard = 2048  # bf16 elements = 4 KB
    n = N * H * W * C
    buf = torch.full((guard + n + guard,), float("nan"), device="cuda", dtype=torch.bfloat16)
    sentinel = buf[:1].view(torch.int16).clone()
    y = buf[guard:guard + n]
    native.check(native.load().vqb_gn_silu_apply(x.data_ptr(), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                                 mr.data_ptr(), N, H * W, C, 32, 1, native.stream_ptr()),
                 "gn_silu_apply")
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), y_ref.reshape(-1).view(torch.int16))
    assert bool((buf[:guard].view(torch.int16) == sentinel).all())
    assert bool((buf[guard + n:].view(torch.int16) == sentinel).all())


# ------------------------------------------------------------------------------------------------ block
def _block(cin, cout, seed=0):
    import ae

    torch.manual_seed(seed)
    blk = ae.ResnetBlock(cin, cout).cuda()
    with torch.no_grad():
        blk.conv2.weight.normal_(0, 0.05)  # the reference's near-zero conv2 init would hide the residual branch
        for p in (blk.norm1.bias, blk.norm2.bias, blk.conv1.bias, blk.conv2.bias):
            p.normal_(0, 0.1)
    return blk


def _act(x_nchw):
    """-> Act of x with the column sums the producing conv's epilogue would hand over."""
    import ae
    import ops

    t = ops.to_nhwc(x_nchw.detach())
    tf = t.float()
    st = torch.stack([tf.sum((1, 2)), tf.pow(2).sum((1, 2))], -1).contiguous()
    return ae.Act(t, x_nchw.shape[1], st)


# (cin, cout, H, W): conv1 fuses the statistics at 16x32; not at 20x24 (ragged pixel tiles)
@pytest.mark.parametrize("cin,cout,H,W,fused", [(64, 128, 16, 32, True), (128, 128, 20, 24, False),
                                                (128, 64, 20, 24, False), (128, 128, 16, 32, True)])
def test_block_forward_matches_the_plain_forward(cin, cout, H, W, fused):
    import ae

    blk = _block(cin, cout)
    a = _act(torch.randn(2, cin, H, W, device="cuda"))

    def fwd(recompute):
        ae.enable_recompute(blk, recompute)
        o = blk(ae.Act(a.t, a.C, a.stats))
        return o.t.detach().clone(), o.stats

    plains = [fwd(False) for _ in range(3)]
    rec = fwd(True)
    assert (rec[1] is None) == (plains[0][1] is None) == (not fused)
    if not fused:
        assert all(torch.equal(_bits(p[0]), _bits(rec[0])) for p in plains)
    else:
        r = _same_as_plain("block out", rec[0].float(), [p[0].float() for p in plains])
        _same_as_plain("block out stats", rec[1], [p[1] for p in plains])
        print(f"\nResnetBlock({cin}, {cout}) at {H}x{W}: recompute out / plain spread {r}")


@pytest.mark.parametrize("cin,cout,H,W", [(64, 128, 16, 32), (128, 128, 20, 24)])
def test_rebuilt_activations_equal_the_forward(cin, cout, H, W):
    """What the backward rebuilds from the saved x and mr records (GroupNorm apply, conv1 without the statistics
    epilogue, GroupNorm apply) is, bit for bit, what the forward computed: conv2 over the rebuilt h2 (with the skip)
    reproduces the node's output. Where the plain forward is deterministic (no fused statistics at 20x24), the rebuilt
    hn, h and h2 also equal the tensors the plain path saves."""
    import ae
    import ops

    blk = _block(cin, cout)
    a = _act(torch.randn(2, cin, H, W, device="cuda"))
    params = {p.data_ptr() for p in blk.parameters()}
    ae.enable_recompute(blk)
    out = blk(ae.Act(a.t, a.C, a.stats)).t
    x, mr1, mr2 = out.grad_fn.saved_tensors[:3]
    assert x.data_ptr() == a.t.data_ptr()
    with torch.no_grad():
        hn = ops.gn_silu_apply(x, blk.norm1.weight, blk.norm1.bias, mr1, True)
        h = ops.conv(hn, blk.conv1.weight, blk.conv1.bias, blk.conv1._packed, "s1")
        h2 = ops.gn_silu_apply(h, blk.norm2.weight, blk.norm2.bias, mr2, True)
        skip = blk.nin_shortcut.forward_act(ae.Act(x, cin)).t if cin != cout else x
        again = ops.conv(h2, blk.conv2.weight, blk.conv2.bias, blk.conv2._packed, "s1", residual=skip)
    assert torch.equal(_bits(again), _bits(out))
    if (H, W) == (20, 24):
        ae.enable_recompute(blk, False)
        plain = [t for t in _saved(lambda: blk(ae.Act(a.t, a.C, a.stats)))[0] if t.data_ptr() not in params]
        # saved by the plain path in this order: x (norm1), mr1, hn (conv1), h (norm2), mr2, [x (nin_shortcut)], h2
        for what, p, r in (("x", plain[0], x), ("mr1", plain[1], mr1), ("hn", plain[2], hn), ("h", plain[3], h),
                           ("mr2", plain[4], mr2), ("h2", plain[-1], h2)):
            assert torch.equal(p.reshape(-1), r.reshape(-1)), what


@pytest.mark.parametrize("cin,cout", [(64, 128), (128, 128)])
def test_saved_tensors_per_block_drop_to_the_input(cin, cout):
    """Counted from the shapes: without recompute a ResnetBlock keeps x, hn, h and h2 (bf16) and two [N, 32, 2] fp32
    GroupNorm records; with recompute, x and the two records. The parameters it saves are its own."""
    import ae

    blk = _block(cin, cout)
    N, H, W = 2, 16, 32
    x = torch.randn(N, cin, H, W, device="cuda", requires_grad=True)
    params = {p.data_ptr(): p for p in blk.parameters()}
    px = N * H * W
    stats = 2 * N * 32 * 2 * 4
    want = {False: 2 * px * (2 * cin + 2 * cout) + stats, True: 2 * px * cin + stats}
    for recompute in (False, True):
        ae.enable_recompute(blk, recompute)
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


def test_weight_changed_in_place_between_forward_and_backward_raises():
    import ae

    blk = ae.enable_recompute(_block(64, 64))
    out = blk(torch.randn(1, 64, 16, 16, device="cuda", requires_grad=True))
    with torch.no_grad():
        blk.conv1.weight.mul_(1.01)
    with pytest.raises(RuntimeError, match="inplace"):
        out.sum().backward()


# ------------------------------------------------------------------------------------------------ module
FLUX_ATTN = VO.VAEConfig(resolution=32, ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=4, use_attn=True)
CONFIGS = {  # name: (config, golden (None: no oracle bounds), input shape, wavelet)
    "vae_attn": (FLUX_ATTN, "vae_attn", (2, 3, 32, 32), False),
    "vae_hr": (VO.VAEConfig(resolution=32, ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=4,
                            decoder_also_perform_hr=True), "vae_hr", (1, 3, 32, 32), False),
    "wavelet": (VO.VAEConfig(resolution=64, ch=32, ch_mult=(1, 2, 2), num_res_blocks=1, z_channels=4), None,
                (2, 3, 64, 64), True),
}


def _make(name):
    import ae

    cfg, gname, shape, wavelet = CONFIGS[name]
    if wavelet:
        torch.manual_seed(11)
        m = ae.VAE(resolution=cfg.resolution, in_channels=3, ch=cfg.ch, out_ch=3, ch_mult=list(cfg.ch_mult),
                   num_res_blocks=cfg.num_res_blocks, z_channels=cfg.z_channels, use_attn=False,
                   decoder_also_perform_hr=False, use_wavelet=True).cuda()
    else:
        m = build_vae(cfg, gname)
    x = seeded.tensor(f"{gname or name}/x", shape, 1.0, "uniform").cuda()
    return m, x


def _step(m, x, recompute):
    """One forward + backward of the parity tests' loss -> ({name: grad}, grad of x)."""
    import ae

    ae.enable_recompute(m, recompute)
    m.zero_grad(set_to_none=True)
    xi = x.clone().requires_grad_(True)
    dec, z = m(xi)
    (dec.pow(2).mean() + z.pow(2).mean()).backward()
    torch.cuda.synchronize()
    return {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}, xi.grad


@pytest.mark.parametrize("name", list(CONFIGS))
def test_recompute_gradients_match_the_plain_path(name):
    m, x = _make(name)
    plains = [_step(m, x, False) for _ in range(3)]
    rg, rx = _step(m, x, True)
    _check_grads_same(name, rg, [p[0] for p in plains])
    _same_as_plain(f"{name} input grad", rx, [p[1] for p in plains])
    gname = CONFIGS[name][1]
    if gname is not None:  # the oracle bounds of test_gpu_parity.py, on the recompute gradients
        g = golden(gname)
        params = dict(m.named_parameters())
        for k, p in params.items():
            p.grad = rg.get(k)
        check_grads(m.named_parameters(), g)
        for k in g:
            if k.startswith("grad::"):
                assert cosine(params[k[6:]].grad, g[k]) > COS_TOL, k


def test_recompute_adds_exactly_conv1_and_two_groupnorm_applies_per_block():
    """native.launch_count() of a recompute step minus a plain step = (one conv1 launch + two GroupNorm apply launches)
    per ResnetBlock: no extra column sum or statistics pass."""
    import native

    m, x = _make("vae_attn")
    for rc in (False, True):  # warm-up: packs every forward and transposed operand
        _step(m, x, rc)

    def count(recompute):
        torch.cuda.synchronize()
        n0 = native.launch_count()
        _step(m, x, recompute)
        return native.launch_count() - n0

    plain, rec = count(False), count(True)
    nblocks = len(_blocks(m))
    print(f"\nlaunches per step: plain {plain}, recompute {rec}, {nblocks} ResnetBlocks")
    assert rec - plain == nblocks * (1 + 2)


# peak allocated memory of a forward + backward of the FLUX config (ch=128, ch_mult 1,2,4,4, two blocks per level) at
# 256^2, batch 4, with recompute over without. Measured on an H100 80GB HBM3 at a 700 W power limit: 1.22 GiB against
# 2.85 GiB, a ratio of 0.427. The bound leaves a margin of 0.073 for allocator and transient-buffer variation.
MEMORY_RATIO_BOUND = 0.5


def test_recompute_lowers_peak_memory():
    import ae

    torch.manual_seed(1)
    m = ae.VAE(resolution=256, in_channels=3, ch=128, out_ch=3, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
               z_channels=16, use_attn=False, decoder_also_perform_hr=False, use_wavelet=False).cuda()
    x = torch.rand(4, 3, 256, 256, device="cuda") * 2 - 1

    def peak(recompute):
        ae.enable_recompute(m, recompute)
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        dec, z = m(x)
        (dec.pow(2).mean() + z.pow(2).mean()).backward()
        del dec, z
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    peak(False)  # packs the weights, plans the shapes
    plain, rec = peak(False), peak(True)
    print(f"\npeak allocated, forward + backward of the FLUX config at 256^2, batch 4: plain {plain / 2 ** 30:.2f} GiB, "
          f"recompute {rec / 2 ** 30:.2f} GiB, ratio {rec / plain:.3f}")
    assert rec <= MEMORY_RATIO_BOUND * plain


def test_bf16_module_with_the_flag_is_unchanged_and_refuses_the_backward():
    import ae

    m, x = _make("vae_attn")
    m = m.bfloat16()
    xb = x.bfloat16()
    with torch.no_grad():
        plain = m(xb)
        ae.enable_recompute(m)
        rec = m(xb)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(plain, rec))
    errors = []
    for recompute in (False, True):
        ae.enable_recompute(m, recompute)
        dec, z = m(xb)
        with pytest.raises(RuntimeError, match="bf16 modules are inference-only") as e:
            (dec.float().pow(2).mean() + z.float().pow(2).mean()).backward()
        errors.append(str(e.value))
    assert errors[0] == errors[1]
    blk = ae.enable_recompute(_block(64, 64).bfloat16())  # the node's own guard
    out = blk(torch.randn(1, 64, 16, 16, device="cuda", dtype=torch.bfloat16))
    assert out.grad_fn is not None
    with pytest.raises(RuntimeError, match="bf16 modules are inference-only"):
        out.float().sum().backward()


# ------------------------------------------------------------------------------------------------ Trainer
def _trainer_run(recompute, graph, steps=8, **kw):
    import random

    import vae_trainer as vt

    args = dict(vae_resolution=64, vae_ch=32, vae_ch_mult="1,2", vae_num_res_blocks=1, vae_z_channels=4,
                do_clamp=True, do_ganloss=True, disc_type="hinge", use_lecam=True, max_steps=50,
                learning_rate_vae=2e-2, lpips_eval=True)
    args.update(kw)
    res = 512 if args.get("decoder_also_perform_hr") else 256
    tr = vt.Trainer("cuda:0", cuda_graph=graph, recompute=recompute, **args)
    random.seed(123)
    g = torch.Generator().manual_seed(9)
    batches = [(torch.rand(2, 3, res, res, generator=g) * 2 - 1).pin_memory() for _ in range(3)]
    losses = [float(tr.step(batches[i % 3])["overall_vae_loss"]) for i in range(steps)]
    torch.cuda.synchronize()
    w = tr.vae.module.decoder.conv_out.weight.detach().float().clone()
    tr.release_graph()
    return tr, losses, w


def test_trainer_recompute_graph_matches_eager_and_tracks_the_plain_losses():
    """Trainer(recompute=True): the CUDA-graph replayed trajectory (GAN + LeCam + GradNorm) equals the eager one within
    the tolerance of test_gpu_train.py's graph-vs-eager test, and its eight losses follow the plain Trainer's within the
    plain runs' own spread."""
    tr_e, le, we = _trainer_run(True, False)
    tr_g, lg, wg = _trainer_run(True, True)
    assert tr_e.graph_launches_per_step is None
    for a, b in zip(le, lg):
        assert abs(a - b) <= 2e-2 * max(abs(a), 0.05), (le, lg)
    assert rel_l2(wg, we) < 2e-2
    plains = [torch.tensor(_trainer_run(False, True)[1], dtype=torch.float64) for _ in range(3)]
    print(f"\nplain losses     {['%.5f' % v for v in plains[0].tolist()]}\nrecompute losses "
          f"{['%.5f' % v for v in lg]}")
    _same_as_plain("Trainer loss curve", torch.tensor(lg, dtype=torch.float64), plains)


@pytest.mark.parametrize("kw", [dict(use_vq=True), dict(decoder_also_perform_hr=True), dict(use_wavelet=True)],
                         ids=["vq", "hr", "wavelet"])
def test_trainer_recompute_runs_the_gan_vq_hr_and_wavelet_configs(kw):
    tr, losses, w = _trainer_run(True, True, steps=5, **kw)
    assert all(np.isfinite(losses))
    assert all(b._vqb_recompute for b in _blocks(tr.vae.module))
