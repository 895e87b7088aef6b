"""GPU (-m gpu): no-grad fp32 / bf16 inference of the video autoencoder (tae.TVAE) on the native kernels.

Tolerance rule (as in test_gpu_infer.py). Truth is oracle/tae_oracle.py run in fp32 on this GPU (TF32 off) with the
SAME bf16-rounded weights and input. The peer is the same oracle in bf16 with cuDNN. Our error must satisfy
rel_L2(ours) <= 1.5 x rel_L2(peer) + FLOOR.
"""
import pytest
import torch
import torch.nn.functional as F

from helpers import golden, rel_l2, t
from oracle import seeded
from oracle import tae_oracle as TO

pytestmark = pytest.mark.gpu

FLOOR = 2e-3
SMALL = TO.TAEConfig(ch=32, ch_mult=(1, 8), num_res_blocks=1, z_channels=4, resolution=16)


class tf32_off:
    def __enter__(self):
        self.s = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.s


def check(what, ours, truth, peer, dtype=None):
    if dtype is not None:
        assert ours.dtype == dtype, (what, ours.dtype)
    assert ours.shape == truth.shape == peer.shape, (what, ours.shape, truth.shape)
    assert bool(torch.isfinite(ours.float()).all()), what
    e, p = rel_l2(ours, truth), rel_l2(peer, truth)
    print(f"\n{what}: ours rel {e:.3e}  bf16 cuDNN peer rel {p:.3e}  (vs fp32 truth)")
    assert e <= 1.5 * p + FLOOR, (what, e, p)
    return e, p


def make_tvae(cfg, tag, dtype):
    """-> (our TVAE with seeded bf16-rounded weights in `dtype` on cuda, the fp32 state_dict holding those values)."""
    import tae

    m = tae.TVAE(**cfg.kwargs())
    sd = {k: v.bfloat16().float() for k, v in seeded.fill_state_dict(m.state_dict(), tag).items()}
    m.load_state_dict(sd)
    return m.cuda().to(dtype).eval(), sd


def arms(fn, sd, *inps):
    """-> (fp32 truth, bf16 cuDNN peer) of fn(state_dict, *inputs) on the GPU."""
    with torch.no_grad(), tf32_off():
        truth = fn({k: v.cuda() for k, v in sd.items()}, *[i.float().cuda() for i in inps])
        peer = fn({k: v.cuda().bfloat16() for k, v in sd.items()}, *[i.bfloat16().cuda() for i in inps])
    return truth, peer


# ------------------------------------------------------------------------------------------------ kernel level
def _nthwc(x):
    import ops

    N, C, T, H, W = x.shape
    y = ops.to_nhwc(x.reshape(N, C, T * H, W))
    return y.view(N, T, H, W, y.shape[-1])


def _ncthw(y, C):
    N, T, H, W, Cp = y.shape
    return y[..., :C].permute(0, 4, 1, 2, 3).float()


@pytest.mark.parametrize("kind", ["s1", "s2", "up"])
@pytest.mark.parametrize("Cout", [3, 16, 64, 256])
def test_conv3d_kernel_matches_conv3d(kind, Cout):
    import ops

    g = torch.Generator(device="cuda").manual_seed(Cout)
    C = 8
    T, H, W = (6, 10, 22) if kind == "s2" else (5, 9, 21)  # ragged tiles; s2 needs even extents
    x = (torch.rand(2, C, T, H, W, device="cuda", generator=g) - 0.5).bfloat16().float()
    w = (torch.randn(Cout, C, 3, 3, 3, device="cuda", generator=g) * 0.2).bfloat16().float()
    b = torch.randn(Cout, device="cuda", generator=g) * 0.1
    xa = _nthwc(x)
    cache = ops.PackedCache()

    def ref(w_, x_, b_):
        if kind == "s1":
            return F.conv3d(x_, w_, b_.to(x_.dtype), padding=1)
        if kind == "s2":
            return F.conv3d(F.pad(x_, (0, 1, 0, 1, 0, 1)), w_, b_.to(x_.dtype), stride=2)
        return F.conv3d(F.interpolate(x_, scale_factor=2.0, mode="nearest"), w_, b_.to(x_.dtype), padding=1)

    with torch.no_grad():
        with tf32_off():
            truth, peer = ref(w, x, b), ref(w.bfloat16(), x.bfloat16(), b)
        To, Ho, Wo = truth.shape[2:]
        if kind == "up":
            ours = _ncthw(ops.upsample_conv3d(xa, w, b, cache), Cout)
            check(f"up Cout={Cout}", ours, truth, peer)
            return
        ours = _ncthw(ops.conv3d(xa, w, b, cache, kind), Cout)
        check(f"{kind} Cout={Cout} NTHWC bf16", ours, truth, peer)
        # bias + residual (bf16, in the output's layout), NTHWC store and strided NCTHW module-boundary stores in fp32
        # and bf16
        r = (torch.rand(2, Cout, To, Ho, Wo, device="cuda", generator=g) - 0.5).bfloat16().float()
        ours = _ncthw(ops.conv3d(xa, w, b, cache, kind, residual=_nthwc(r)), Cout)
        check(f"{kind} Cout={Cout} NTHWC bf16 +res", ours, truth + r, peer + r.bfloat16())
        for wd in (torch.float32, torch.bfloat16):
            o = ops.conv3d(xa, w.to(wd), b, ops.PackedCache(), kind, residual=r.bfloat16(), ncthw_out=True)
            assert o.dtype == wd and o.shape == (2, Cout, To, Ho, Wo)
            check(f"{kind} Cout={Cout} NCTHW {wd} +res", o, truth + r, peer + r.bfloat16())


@pytest.mark.parametrize("head_dim", [32, 64])
def test_attention_heads_match_sdpa(head_dim):
    import ops

    g = torch.Generator(device="cuda").manual_seed(head_dim)
    N, T, heads = 2, 6144, 8
    C = heads * head_dim
    qkv = (torch.randn(N, 6, 32, 32, 3 * C, device="cuda", generator=g)).bfloat16()
    with torch.no_grad():
        ours = ops.attention_hd(qkv, heads, head_dim).reshape(N, T, heads, head_dim).permute(0, 2, 1, 3)
        q, k, v = (u.reshape(N, T, heads, head_dim).permute(0, 2, 1, 3) for u in qkv.reshape(N, T, 3 * C).chunk(3, -1))
        with tf32_off():
            truth = F.scaled_dot_product_attention(q.float(), k.float(), v.float())
        peer = F.scaled_dot_product_attention(q, k, v)
    check(f"attention heads of {head_dim}", ours, truth, peer, torch.bfloat16)


# ------------------------------------------------------------------------------------------------ module parity
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_golden_config_matches_oracle_and_reference(dtype):
    import ops

    gd = golden("tae_small")
    m, sd = make_tvae(SMALL, "tae_small", dtype)
    x, eps = t(gd["x"]).bfloat16().float(), t(gd["eps"])
    with torch.no_grad():
        z = m.encoder(x.cuda().to(dtype))
        decz = m.decoder(ops.gauss_reparam(z, eps.cuda().to(dtype)))
    tz, pz = arms(lambda s, x_: TO.encoder_forward(s, x_, SMALL), sd, x)
    td, pd = arms(lambda s, x_, e_: TO.forward(s, x_, e_, SMALL)[0], sd, x, eps)
    check(f"tae_small z {dtype}", z, tz, pz, dtype)
    check(f"tae_small decz {dtype}", decz, td, pd, dtype)
    assert z.shape == gd["z"].shape and decz.shape == gd["decz"].shape
    # against the reference's own fp32 result (unrounded weights and input): within the same rule plus the effect of
    # rounding the weights and input to bf16, which the fp32 truth also carries
    assert rel_l2(decz.float().cpu(), gd["decz"]) <= 1.5 * rel_l2(pd.float().cpu(), gd["decz"]) + \
        rel_l2(td.cpu(), gd["decz"]) + FLOOR
    assert rel_l2(z.float().cpu(), gd["z"]) <= 1.5 * rel_l2(pz.float().cpu(), gd["z"]) + rel_l2(tz.cpu(), gd["z"]) + FLOOR


def encode_decode_parity(what, cfg, m, sd, x, eps, dtype):
    """Encoder on x, decoder on one common latent: the fp32 truth's sampled latent rounded to bf16 (the decoder amplifies
    a difference in its input, so each half is held to the rule on the same input)."""
    with torch.no_grad():
        z = m.encoder(x.cuda().to(dtype))
    tz, pz = arms(lambda s, x_: TO.encoder_forward(s, x_, cfg), sd, x)
    check(f"{what} z {dtype}", z, tz, pz, dtype)
    zshape = tuple(z.shape)
    zs = TO.reg(tz, eps.cuda()).bfloat16().float()
    del z, tz, pz
    with torch.no_grad():
        decz = m.decoder(zs.to(dtype))
    td, pd = arms(lambda s, z_: TO.decoder_forward(s, z_, cfg), sd, zs)
    check(f"{what} decz {dtype}", decz, td, pd, dtype)
    return zshape, tuple(decz.shape)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_heads_of_64_config(dtype):
    cfg = TO.TAEConfig(ch=128, ch_mult=(1, 4), num_res_blocks=1, z_channels=4, resolution=64)
    m, sd = make_tvae(cfg, "tae_h64", dtype)
    assert m.encoder.mid.attn_1.head_dim == 64
    x = seeded.tensor("tae_h64/x", (2, 3, 8, 64, 96), 1.0, "uniform").bfloat16().float()
    eps = seeded.tensor("tae_h64/eps", (2, 4, 4, 32, 48), 1.0)
    encode_decode_parity("heads-of-64", cfg, m, sd, x, eps, dtype)


def test_reference_main_config_bf16():
    """tae.py's __main__: ch=64, ch_mult [1,2,4,4], num_res_blocks 2, z_channels 16 on (1, 3, 48, 256, 256)."""
    cfg = TO.TAEConfig()
    m, sd = make_tvae(cfg, "tae_main", torch.bfloat16)
    assert m.encoder.mid.attn_1.head_dim == 32
    x = seeded.tensor("tae_main/x", (1, 3, 48, 256, 256), 1.0, "uniform").bfloat16().float()
    eps = seeded.tensor("tae_main/eps", (1, 16, 6, 32, 32), 1.0)
    zshape, dshape = encode_decode_parity("main config", cfg, m, sd, x, eps, torch.bfloat16)
    assert zshape == (1, 32, 6, 32, 32) and dshape == (1, 3, 48, 256, 256)


# ------------------------------------------------------------------------------------------------ sampling
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_sampling_draws_the_reference_noise(dtype):
    import ops

    m, sd = make_tvae(SMALL, "tae_small", dtype)
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").cuda().to(dtype)
    with torch.no_grad():
        torch.manual_seed(11)
        decz, z = m(x)
        torch.manual_seed(11)
        eps = torch.randn_like(z.chunk(2, dim=1)[0])  # the reference's call, same seed
        assert torch.equal(m.decoder(ops.gauss_reparam(z, eps)), decz)
        # the oracle fed with that eps
        td, pd = arms(lambda s, z_, e_: TO.decoder_forward(s, TO.reg(z_, e_), SMALL), sd, z.float(), eps.float())
        check(f"sampled decz {dtype}", decz, td, pd, dtype)
        # the reparameterisation kernel against the fp32 formula: within one rounding of the module's dtype
        zs = ops.gauss_reparam(z, eps)
        ref = TO.reg(z.double(), eps.double())
        mean, logvar = z.double().chunk(2, dim=1)
        scale = mean.abs() + (torch.exp(0.5 * logvar.clamp(min=-3)) * eps.double()).abs()
        ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -21
        assert bool(((zs.double() - ref).abs() <= ulp * scale).all())
        # sample=False returns mean bit for bit
        m.reg.sample = False
        assert torch.equal(m.reg(z), z[:, :SMALL.z_channels])


# ------------------------------------------------------------------------------------------------ determinism
def test_graph_replay_and_second_eager_run_are_bit_identical():
    m, _ = make_tvae(SMALL, "tae_small", torch.bfloat16)
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").cuda().bfloat16()

    def run():
        z = m.encoder(x)
        return z, m.decoder(z[:, :SMALL.z_channels].contiguous())

    with torch.no_grad():
        a = run()
        b = run()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = run()
        graph.replay()
        torch.cuda.synchronize()
    for u, v, w in zip(a, b, static):
        assert torch.equal(u, v) and torch.equal(u, w)


def test_weight_updates_repack_the_27_tap_operands():
    """load_state_dict (version bump) and ops.weights_updated (in-place .data writes) re-pack 3x3x3 weights, which take
    the per-tensor pack kernels."""
    import ops
    import tae

    m, sd = make_tvae(SMALL, "tae_small", torch.float32)
    x = seeded.tensor("tae_small/x", (1, 3, 4, 16, 24), 1.0, "uniform").cuda()
    sd2 = {k: v.bfloat16().float() for k, v in seeded.fill_state_dict(sd, "tae_small/2").items()}
    fresh = tae.TVAE(**SMALL.kwargs())
    fresh.load_state_dict(sd2)
    fresh = fresh.cuda().eval()
    with torch.no_grad():
        m.encoder(x)
        m.load_state_dict(sd2)
        z1 = m.encoder(x)
        zf = fresh.encoder(x)
        assert torch.equal(z1, zf)
        w = m.encoder.conv_in.weight
        w.data.copy_(torch.flip(w.data, dims=[2]))
        ops.weights_updated()
        z2 = m.encoder(x)
        fresh.encoder.conv_in.weight.data.copy_(w.data)
        ops.weights_updated()
        assert torch.equal(z2, fresh.encoder(x)) and not torch.equal(z2, z1)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing():
    import native

    m, _ = make_tvae(SMALL, "tae_small", torch.float32)
    x = torch.zeros(1, 3, 4, 16, 24, device="cuda")
    n0 = native.launch_count()
    with pytest.raises(RuntimeError, match="no_grad"):
        m(x)
    with torch.no_grad(), pytest.raises(ValueError, match=r"\(1, 3, 4, 16, 23\)"):
        m(torch.zeros(1, 3, 4, 16, 23, device="cuda"))
    with torch.no_grad(), pytest.raises(ValueError, match="even"):
        m.encoder.down[0].downsample(torch.zeros(1, 32, 3, 16, 24, device="cuda"))
    h = m.half()
    with torch.no_grad(), pytest.raises(RuntimeError, match="float16"):
        h(x.half())
    torch.cuda.synchronize()
    assert native.launch_count() == n0
