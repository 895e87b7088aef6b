"""GPU (-m gpu): no-grad bf16 / fp32 inference through the drop-in modules (the reference model card's recipe:
`VAE(...).cuda().bfloat16()`, `z = vae.encoder(img).clamp(-8, 8)`, `decz = vae.decoder(z)`).

Tolerance rule. Truth is the CPU-oracle arithmetic (oracle/vae_oracle.py, pinned to the reference) run in fp32 on this
GPU (TF32 off) with the SAME bf16-rounded weights and input. The peer is the model card's own arithmetic: the same
oracle in bf16 with cuDNN, no autocast. Our error must satisfy err_ours <= 1.5 x err_peer + FLOOR (relative L2).
"""
import numpy as np
import pytest
import torch

from helpers import golden, rel_l2
from oracle import lpips_oracle as LP
from oracle import seeded
from oracle import vae_oracle as VO

pytestmark = pytest.mark.gpu

FLOOR = 2e-3


def make_vae(cfg: VO.VAEConfig, tag, dtype, use_wavelet=False):
    """Our VAE with seeded weights (seeded.fill_state_dict of its own state_dict), converted to `dtype` on cuda.
    -> (module, fp32 state_dict holding the bf16-rounded weights every arm uses)."""
    import ae

    m = ae.VAE(resolution=cfg.resolution, in_channels=3, ch=cfg.ch, out_ch=3, ch_mult=list(cfg.ch_mult),
               num_res_blocks=cfg.num_res_blocks, z_channels=cfg.z_channels, use_attn=cfg.use_attn,
               decoder_also_perform_hr=False, use_wavelet=use_wavelet)
    sd = {k: v.bfloat16().float() for k, v in seeded.fill_state_dict(m.state_dict(), tag).items()}
    m.load_state_dict(sd)
    return m.cuda().to(dtype).eval(), sd


class tf32_off:
    def __enter__(self):
        self.s = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.s


def oracle_arms(fn, sd, inp):
    """-> (fp32 truth, bf16 cuDNN peer) of fn(state_dict, input) on the GPU."""
    with torch.no_grad(), tf32_off():
        truth = fn({k: v.cuda() for k, v in sd.items()}, inp.float().cuda())
        peer = fn({k: v.cuda().bfloat16() for k, v in sd.items()}, inp.bfloat16().cuda())
    return truth, peer


def check(what, ours, truth, peer, dtype):
    assert ours.dtype == dtype, (what, ours.dtype)
    assert peer.dtype == torch.bfloat16 and ours.shape == truth.shape
    e, p = rel_l2(ours, truth), rel_l2(peer, truth)
    print(f"\n{what}: ours rel {e:.3e}  eager bf16 cuDNN peer rel {p:.3e}  (vs fp32 truth)")
    assert bool(torch.isfinite(ours.float()).all())
    assert e <= 1.5 * p + FLOOR, (what, e, p)
    return e, p


def encode_decode_parity(cfg, tag, shape, dtype=torch.bfloat16):
    vae, sd = make_vae(cfg, tag, dtype)
    x = seeded.tensor(tag + "/x", shape, 1.0, "uniform").bfloat16().float()
    with torch.no_grad():
        z = vae.encoder(x.cuda().to(dtype)).clamp(-8.0, 8.0)
    tz, pz = oracle_arms(lambda s, i: VO.encoder_forward(s, i, cfg).clamp(-8.0, 8.0), sd, x)
    check(f"{tag} encode {tuple(shape)}", z, tz, pz, dtype)
    zin = tz.bfloat16().float()  # every decoder arm decodes the same latent
    with torch.no_grad():
        dec = vae.decoder(zin.to(dtype))
    td, pd = oracle_arms(lambda s, i: VO.decoder_forward(s, i, cfg), sd, zin)
    check(f"{tag} decode {tuple(zin.shape)}", dec, td, pd, dtype)
    return z, dec


GOLDEN_CFG = VO.VAEConfig(resolution=32, ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=4, use_attn=True)


def test_bf16_inference_vs_reference_golden():
    """The reference's own bf16 model-card run (tests/golden/infer_bf16_attn.npz) on the same bf16 weights."""
    g = golden("infer_bf16_attn")
    vae, sd = make_vae(GOLDEN_CFG, "infer_bf16_attn", torch.bfloat16)
    x = torch.from_numpy(g["x"]).cuda().bfloat16()
    with torch.no_grad():
        z = vae.encoder(x).clamp(-8.0, 8.0)
        dec = vae.decoder(z)
    assert z.dtype == dec.dtype == torch.bfloat16
    tz, pz = oracle_arms(lambda s, i: VO.encoder_forward(s, i, GOLDEN_CFG).clamp(-8.0, 8.0), sd, x)
    check("golden cfg encode", z, tz, pz, torch.bfloat16)
    td, pd = oracle_arms(lambda s, i: VO.decoder_forward(s, i, GOLDEN_CFG), sd, z.float())
    check("golden cfg decode", dec, td, pd, torch.bfloat16)
    ez, ed = rel_l2(z, g["z"]), rel_l2(dec, g["dec"])
    gz, gd = rel_l2(torch.from_numpy(g["z"]), tz), rel_l2(torch.from_numpy(g["dec"]), td)
    print(f"  vs the reference bf16 golden: z rel {ez:.3e} dec rel {ed:.3e} (golden vs fp32 truth: {gz:.3e} {gd:.3e})")
    # two bf16 implementations, each a few 1e-3 .. 1e-2 from the fp32 truth
    assert ez <= 1.5 * gz + rel_l2(z, tz) + FLOOR and ed <= 1.5 * gd + rel_l2(dec, td) + FLOOR


def test_model_card_config_768_bf16():
    """README.hf.md "How to use": ch=256, ch_mult 1,2,4,4, z=16, use_attn=True, 768x768, B=1 (9216 attention tokens)."""
    cfg = VO.VAEConfig(resolution=256, ch=256, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=16, use_attn=True)
    z, dec = encode_decode_parity(cfg, "infer/card", (1, 3, 768, 768))
    assert z.shape == (1, 16, 96, 96) and dec.shape == (1, 3, 768, 768)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_flux_config_768x512_b4(dtype):
    cfg = VO.VAEConfig(resolution=256, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=16)
    z, dec = encode_decode_parity(cfg, "infer/flux", (4, 3, 768, 512), dtype)
    assert z.shape == (4, 16, 96, 64) and dec.shape == (4, 3, 768, 512)


@pytest.mark.parametrize("hw", [(768, 768), (768, 512), (1024, 1024)])
def test_small_attention_model_sizes(hw):
    cfg = VO.VAEConfig(resolution=256, ch=32, ch_mult=(1, 2, 4, 4), num_res_blocks=1, z_channels=4, use_attn=True)
    z, dec = encode_decode_parity(cfg, "infer/small", (1, 3) + hw)
    assert z.shape == (1, 4, hw[0] // 8, hw[1] // 8) and dec.shape == (1, 3) + hw


def _wavelet_encoder_forward(sd, x, mult, nrb):
    """ae.py Encoder with use_wavelet=True (utils.py:229-247 front-end, no Downsample after level 0); `mult` is the
    encoder's ch_mult after the constructor doubled its first entry."""
    p = "encoder"
    h = VO.conv(sd, p + ".conv_in", LP.wavelet_transform_multi_channel(x))
    for i in range(len(mult)):
        for j in range(nrb):
            h = VO.resnet_block(sd, f"{p}.down.{i}.block.{j}", h)
        if i != len(mult) - 1 and i != 0:
            h = VO.downsample(sd, f"{p}.down.{i}.downsample", h)
    h = VO.resnet_block(sd, p + ".mid.block_1", h)
    h = VO.resnet_block(sd, p + ".mid.block_2", h)
    return VO.conv(sd, p + ".conv_out", VO.swish(VO.group_norm(sd, p + ".norm_out", h)))


def test_wavelet_model_bf16_encode():
    cfg = VO.VAEConfig(resolution=64, ch=64, ch_mult=(1, 2, 2), num_res_blocks=1, z_channels=8)
    vae, sd = make_vae(cfg, "infer/wavelet", torch.bfloat16, use_wavelet=True)
    x = seeded.tensor("infer/wavelet/x", (2, 3, 64, 96), 1.0, "uniform").bfloat16().float()
    with torch.no_grad():
        z = vae.encoder(x.cuda().bfloat16())
        dec = vae.decoder(z)
    mult = (2, 2, 2)
    tz, pz = oracle_arms(lambda s, i: _wavelet_encoder_forward(s, i, mult, 1), sd, x)
    check("wavelet encode", z, tz, pz, torch.bfloat16)
    assert dec.dtype == torch.bfloat16 and dec.shape == (2, 3, 64, 96)


def test_attention_core_long_sequence_vs_sdpa():
    """The mid-block attention at the model card's 768x768 (T = 96*96 = 9216, C = 1024, 16 heads) vs
    F.scaled_dot_product_attention in fp32 on the same bf16 inputs."""
    import attention
    import torch.nn.functional as F

    torch.manual_seed(0)
    N, H, W, C = 1, 96, 96, 1024
    qkv = (torch.randn(N, H, W, 3 * C, device="cuda") * 0.7).to(torch.bfloat16)
    with torch.no_grad():
        out = attention.mhsa(qkv, C // 64, 64)
        q, k, v = qkv.float().reshape(N, H * W, 3, C // 64, 64).permute(2, 0, 3, 1, 4)
        ref = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(N, H, W, C)
    e = rel_l2(out, ref)
    print(f"\nattn T={H * W} C={C}: out rel {e:.3e}")
    assert out.dtype == torch.bfloat16 and e < 1e-2


def test_bf16_master_packing_is_bit_exact():
    """Packing from a bf16 master equals packing the same values from fp32: plain, dgrad (transposed + rotated), folded
    up-sample taps, the fat-pixel [R][3][64] layout, and the one-launch multi-pack with mixed master dtypes."""
    import ops

    torch.manual_seed(0)
    cases = [((64, 32, 3, 3), list(range(9)), False, 32, False),
             ((64, 32, 3, 3), list(range(8, -1, -1)), True, 64, False),
             ((40, 24, 1, 1), [0], False, 24, False),
             ((48, 40, 3, 3), [0b11011, 0b110110, 0b11011000, 0b110110000], False, 40, True),
             ((48, 40, 3, 3), [0b1, 0b11, 0b110, 0b100, 0b1001, 0b11011, 0b110110, 0b100100, 0b1000, 0b11000,
                               0b110000, 0b100000, 0b1000000, 0b11000000, 0b110000000, 0b100000000], True, 48, True)]
    ents = []
    for shape, tm, tr, kp, fold in cases:
        wb = torch.randn(shape, device="cuda").bfloat16()
        wf = wb.float()
        a, b = ops.pack_weights(wb, tm, tr, kp, fold), ops.pack_weights(wf, tm, tr, kp, fold)
        assert torch.equal(a, b), (shape, tr, fold)
        if not fold and not tr:  # the plain re-layout of a bf16 master is a copy of its values
            assert torch.equal(a[:, :, :shape[1]], wb.reshape(shape[0], shape[1], -1)[:, :, tm].permute(0, 2, 1))
        ents += [(ops._new_pack_entry(wb, tm, tr, kp, fold), b, wb), (ops._new_pack_entry(wf, tm, tr, kp, fold), b, wf)]
    ops._run_pack([e for e, _, _ in ents])
    for e, ref, _ in ents:
        assert torch.equal(e.out, ref)
    wb = torch.randn(64, 3, 3, 3, device="cuda").bfloat16()
    fat = [ops.PackedCache().get(w, ("fat",), list(range(9)), False, 8, fat=True) for w in (wb, wb.float())]
    assert torch.equal(fat[0], fat[1]) and fat[0].shape == (64, 3, 64)


def _small_bf16_vae(tag):
    return make_vae(VO.VAEConfig(resolution=32, ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=4,
                                 use_attn=True), tag, torch.bfloat16)


def test_checkpoint_load_repacks_bf16_model():
    """load_vae_checkpoint (load_state_dict + weights_updated) on a bf16 model that already packed other weights gives
    the outputs of a freshly constructed bf16 model with the loaded weights; fp32 <-> bf16 state dicts load both ways."""
    import vae_trainer as vt

    x = seeded.tensor("infer/ckpt/x", (2, 3, 32, 48), 1.0, "uniform").cuda().bfloat16()
    a, _ = _small_bf16_vae("infer/ckpt/a")
    fresh, sd_b = _small_bf16_vae("infer/ckpt/b")
    import ae

    def packed(m):
        return {(n, k): e.out for n, c in m.named_modules() if isinstance(c, ae.StandardizedC2d)
                for k, e in c._packed._store.items()}

    with torch.no_grad():
        a(x)  # packs a's own weights
        db, zb = fresh(x)
        db2, zb2 = fresh(x)
        assert torch.equal(zb, zb2) and torch.equal(db, db2)  # the no-grad forward is deterministic
        for src in ({k: v.bfloat16() for k, v in sd_b.items()}, sd_b):  # bf16, then fp32 state dict
            vt.load_vae_checkpoint(a, src)
            assert all(p.dtype == torch.bfloat16 for p in a.parameters())
            pa, pf = packed(a), packed(fresh)
            assert pa.keys() == pf.keys() and all(torch.equal(pa[k], pf[k]) for k in pf)  # bit-identical operands
            da, za = a(x)
            print(f"\nreloaded vs fresh: z max|d| {(za.float() - zb.float()).abs().max().item():.3e} "
                  f"dec max|d| {(da.float() - db.float()).abs().max().item():.3e}")
            assert torch.equal(za, zb) and torch.equal(da, db)
        f32, _ = make_vae(GOLDEN_CFG, "infer/ckpt/c", torch.float32)
        f32.load_state_dict(fresh.state_dict())  # bf16 state dict into an fp32 model
        d32, z32 = f32(x.float())
        assert z32.dtype == d32.dtype == torch.float32
        assert rel_l2(z32, zb) < 2e-2 and rel_l2(d32, db) < 2e-2


def test_inference_mode_and_module_dtypes():
    """torch.inference_mode() runs the same path (and keeps the fat-pixel first layer); z / images follow the module
    dtype; DiagonalGaussian and VectorQuantizer follow it too."""
    import ae
    import ops

    vae, _ = _small_bf16_vae("infer/modes")
    x = seeded.tensor("infer/modes/x", (1, 3, 32, 48), 1.0, "uniform").cuda()
    ops._fat_state["ok"] = None  # the first-layer self-check now runs under inference_mode
    with torch.inference_mode():
        d1, z1 = vae(x.bfloat16())
        sub = vae.encoder.down[0].block[0](torch.randn(1, 32, 16, 24, device="cuda").bfloat16())
    assert ops.fat_conv_enabled()
    with torch.no_grad():
        d2, z2 = vae(x.bfloat16())
        zq, loss, idx = ae.VectorQuantizer(n_e=64, e_dim=4).cuda().bfloat16()(z2)
    assert z1.dtype == d1.dtype == sub.dtype == zq.dtype == torch.bfloat16 and idx.shape == (1, 16, 24)
    assert vae.reg(z2).dtype == torch.bfloat16
    assert rel_l2(z1, z2) < 1e-2 and rel_l2(d1, d2) < 1e-2


def test_fp16_module_raises_before_any_launch():
    import native

    vae, _ = _small_bf16_vae("infer/fp16")
    vae = vae.half()
    x = torch.rand(1, 3, 32, 32, device="cuda").half()
    l0 = native.launch_count()
    for fn, arg in ((vae.encoder, x), (vae.decoder, torch.rand(1, 4, 16, 16, device="cuda").half()), (vae, x)):
        with torch.no_grad(), pytest.raises(RuntimeError, match="torch.float16"):
            fn(arg)
    with pytest.raises(RuntimeError, match="torch.float16"):
        vae.encoder.down[0].block[0](torch.rand(1, 32, 16, 16, device="cuda").half())
    assert native.launch_count() == l0


def test_backward_through_bf16_module_raises():
    vae, _ = _small_bf16_vae("infer/bwd")
    x = torch.rand(1, 3, 32, 32, device="cuda").bfloat16()
    z = vae.encoder(x)  # grad enabled: parameters require grad
    with pytest.raises(RuntimeError, match="inference-only"):
        z.float().pow(2).sum().backward()
    dec = vae.decoder(torch.rand(1, 4, 16, 16, device="cuda").bfloat16())
    with pytest.raises(RuntimeError, match="inference-only"):
        dec.float().sum().backward()
    assert all(p.grad is None for p in vae.parameters())


# first H100 run (H100 80GB HBM3, 400 W limit): no-grad 640 MiB vs grad-enabled 3599 MiB above the weights, ratio 5.62;
# the bound keeps a margin below that measurement
MEMORY_RATIO_BOUND = 4.5


def test_no_grad_decode_peak_memory():
    """FLUX config, 256x256, B=8: without autograd the decoder keeps no saved activations alive across blocks."""
    cfg = VO.VAEConfig(resolution=256, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=16)
    vae, _ = make_vae(cfg, "infer/mem", torch.float32)
    z = torch.randn(8, 16, 32, 32, device="cuda")
    with torch.no_grad():
        vae.decoder(z)  # packs the weights, plans the shapes

    def peak(grad):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        with torch.set_grad_enabled(grad):
            out = vae.decoder(z)
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated() - base
        del out
        return p

    ng, g = peak(False), peak(True)
    print(f"\ndecode 8x256x256 peak above weights: no-grad {ng / 2**20:.1f} MiB, grad-enabled {g / 2**20:.1f} MiB, "
          f"ratio {g / ng:.2f}")
    assert g >= MEMORY_RATIO_BOUND * ng


def test_cuda_graph_replay_matches_eager():
    """A no-grad encode + decode captured as one CUDA graph and replayed equals the eager run bit for bit."""
    import ops

    cfg = VO.VAEConfig(resolution=256, ch=64, ch_mult=(1, 2, 4, 4), num_res_blocks=1, z_channels=16, use_attn=True)
    vae, _ = make_vae(cfg, "infer/graph", torch.bfloat16)
    x = seeded.tensor("infer/graph/x", (2, 3, 256, 192), 1.0, "uniform").cuda().bfloat16()

    def run():
        z = vae.encoder(x).clamp(-8.0, 8.0)
        return z, vae.decoder(z)

    assert ops.fat_conv_enabled()
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                run()
        torch.cuda.current_stream().wait_stream(s)
        eager = [run() for _ in range(2)]
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = run()
        graph.replay()
        torch.cuda.synchronize()
    ez, ed = eager[0]
    rz, rd = static
    dz, dd = (rz.float() - ez.float()).abs().max().item(), (rd.float() - ed.float()).abs().max().item()
    nz = (eager[1][0].float() - ez.float()).abs().max().item()
    nd = (eager[1][1].float() - ed.float()).abs().max().item()
    print(f"\ngraph replay vs eager: z max|d| {dz:.3e} dec max|d| {dd:.3e}; eager vs eager: {nz:.3e} {nd:.3e}")
    # without autograd the GroupNorm statistics come from the fixed-order statistics pass, not from the conv epilogue's
    # fp32 atomics (ae._stats_fusion): eager runs and the replay are bit-identical
    assert torch.equal(eager[1][0], ez) and torch.equal(eager[1][1], ed)
    assert torch.equal(rz, ez) and torch.equal(rd, ed)
