"""GPU (-m gpu): the fused PSNR / SSIM kernel (vqb_psnr_ssim via ops.psnr_ssim) and VideoTrainer.evaluate.

Accuracy: every item's PSNR and SSIM against the float64 oracle (oracle/metrics_oracle.py), within a bound derived from
the kernel's fp32 arithmetic on the same inputs (ssim_psnr_bounds below), which must itself be no looser than 1e-3 dB
and 1e-4. Exact cases (identical inputs: +inf and 1.0), memory safety (outputs in sentinel buffers with guard bands,
inputs surrounded by poison), bit-identical reruns, and a float64 F.conv2d cross-check at 2 x 3 x 48 x 256^2.
VideoTrainer.evaluate scores the hand-decoded posterior mean and leaves every piece of trainer state as it was; the
train_video CLI logs eval_psnr, eval_ssim and eval_lpips with --eval_clips.

`python -m pytest -m gpu -q tests/test_gpu_metrics.py -s` prints max(err / bound) per accuracy case.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import seeded_sd
from oracle import lpips_oracle as LP
from oracle import metrics_oracle as MO
from oracle import seeded
from test_gpu_kernel_bounds import BITS, SENTINEL, Guarded, check_bits, check_stores, lib  # noqa: F401
from test_gpu_tae import SMALL, make_tvae

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "vqgan-training_b200")
u = 2.0 ** -24
PSNR_CAP, SSIM_CAP = 1e-3, 1e-4  # the bounds below must never be looser than these

# Rounding counts of the kernel (csrc/metrics.cu), each a first-order count of fp32 roundings of at most u times the
# magnitude named:
#   a = u_x - 0.5                                 1                  of |a|
#   window weights g_i g_j (each g_i rounded)     2                  of w
#   horizontal and vertical 11-tap FMA chains     11 + 11            of sum w |term|
#   product a * b                                 1 (+ 2 from a, b)  of |a b|
N_MU = 1 + 2 + 22    # mu_a = sum w a:              |d mu_a| <= N_MU u sum w |a|
N_SQ = 3 + 2 + 22    # S_ab = sum w a b:            |d S_ab| <= N_SQ u sum w |a b|
N_FORMULA = 12       # the SSIM formula from the five moments: 7 roundings in n1, d1, n2, d2, 3 in the quotient, +2 C1/C2
N_MEAN = 4 + 5 + 8 + 1  # the mean over positions: 4 per thread, 5 shuffle and 8 block levels in fp32, + the fp32 output
N_MSE = 3 + 7 + 5 + 8 + 1  # sum (u_x - u_y)^2: d and d^2 (3), <= 7 terms per thread, 5 shuffle, 8 block levels, + 1
SECOND_ORDER = 2.0   # headroom over the first-order sum for its neglected products of errors


def _planes(v, value_range):
    lo, hi = np.float32(value_range[0]), np.float32(value_range[1])
    inv = float(np.float32(1.0 / (np.float64(hi) - np.float64(lo))))
    v = v if v.dim() == 5 else v.unsqueeze(2)
    v = v.transpose(1, 2).reshape(-1, 1, *v.shape[-2:]).float()
    return ((v - float(lo)) * inv).clamp(0, 1).double()


def ssim_psnr_bounds(x, y, value_range, psnr_ref, ssim_ref):
    """Per-item bounds on |kernel - float64| for PSNR (dB) and SSIM: the first-order propagation of the rounding counts
    above through the SSIM formula at every valid position (partial derivatives in float64), averaged over the item's
    positions, plus the fp32 mean, times SECOND_ORDER."""
    ux, uy = _planes(x, value_range), _planes(y, value_range)
    g = torch.tensor(MO.gaussian_1d(), dtype=torch.float64, device=ux.device)

    def filt(a):
        return F.conv2d(F.conv2d(a, g.view(1, 1, 1, -1)), g.view(1, 1, -1, 1))

    a, b = ux - 0.5, uy - 0.5
    ma, mb = filt(a), filt(b)
    saa, sbb, sab = filt(a * a), filt(b * b), filt(a * b)
    d_ma, d_mb = N_MU * u * filt(a.abs()), N_MU * u * filt(b.abs())
    d_saa, d_sbb, d_sab = N_SQ * u * saa, N_SQ * u * sbb, N_SQ * u * filt((a * b).abs())
    vx, vy, cxy = saa - ma * ma, sbb - mb * mb, sab - ma * mb
    mx, my = ma + 0.5, mb + 0.5
    # the kernel's rounding of the centred variances and of mu + 0.5
    d_vx = d_saa + 2 * ma.abs() * d_ma + u * (ma * ma + vx.abs())
    d_vy = d_sbb + 2 * mb.abs() * d_mb + u * (mb * mb + vy.abs())
    d_cxy = d_sab + mb.abs() * d_ma + ma.abs() * d_mb + u * ((ma * mb).abs() + cxy.abs())
    d_mx, d_my = d_ma + u * mx.abs(), d_mb + u * my.abs()
    n1, d1 = 2 * mx * my + MO.C1, mx * mx + my * my + MO.C1
    n2, d2 = 2 * cxy + MO.C2, vx + vy + MO.C2
    A, Bf = n1 / d1, n2 / d2
    s = A * Bf
    first = (Bf * (2 * my * d1 - 2 * mx * n1).abs() / d1 ** 2 * d_mx + Bf * (2 * mx * d1 - 2 * my * n1).abs() / d1 ** 2
             * d_my + A * n2.abs() / d2 ** 2 * (d_vx + d_vy) + A * 2 / d2 * d_cxy + N_FORMULA * u * s.abs())
    shape = psnr_ref.shape
    n_items = int(np.prod(shape))
    ssim_b = SECOND_ORDER * (first.reshape(n_items, -1).mean(1) + N_MEAN * u * s.abs().reshape(n_items, -1).mean(1))
    psnr_b = SECOND_ORDER * (10 / math.log(10) * N_MSE * u + u * psnr_ref.abs().reshape(-1))
    return psnr_b.view(shape).cpu().numpy(), ssim_b.view(shape).cpu().numpy()


# ---------------------------------------------------------------------------------------------------- inputs
def make_inputs(shape, dtype, value_range, seed):
    """y a noisy copy of x: a ramp over the range plus uniform noise of a per-channel amplitude, so that some values
    lie up to a fifth of the range past either end. Every window keeps some texture (sigma >= ~0.1): in flat windows the
    derived fp32 bound below grows past 1e-4, although the observed error does not."""
    lo, hi = value_range
    gen = torch.Generator(device="cpu").manual_seed(seed)
    H, W = shape[-2:]
    ramp = torch.linspace(0, 1, H).view(H, 1) * 0.3 + torch.linspace(0, 1, W).view(1, W) * 0.3 + 0.2
    amp = torch.tensor([0.8, 0.5, 0.65])[: shape[1]].view(1, -1, *([1] * (len(shape) - 2)))
    x01 = ramp + amp * (torch.rand(shape, generator=gen) - 0.5)
    y01 = x01 + 0.05 * torch.randn(shape, generator=gen)
    x, y = (lo + (hi - lo) * v for v in (x01, y01))
    return x.to(dtype).cuda(), y.to(dtype).cuda()


SIZES = [(11, 11), (11, 40), (12, 12), (33, 67), (67, 129), (256, 256)]
LAYOUTS = ["image", "clip1", "clip5"]


def _shape(layout, C, H, W, B=2):
    return (B, C, H, W) if layout == "image" else (B, C, 1 if layout == "clip1" else 5, H, W)


@pytest.mark.parametrize("value_range", [(0.0, 1.0), (-1.0, 1.0)], ids=["01", "pm1"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("HW", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_accuracy_against_fp64_oracle(HW, C, layout, dtype, value_range):
    import ops

    shape = _shape(layout, C, *HW)
    x, y = make_inputs(shape, dtype, value_range, seed=100 * SIZES.index(HW) + 10 * LAYOUTS.index(layout) + C)
    p, s = ops.psnr_ssim(x, y, value_range=value_range)
    assert p.shape == s.shape == (shape[:1] if layout == "image" else (shape[0], shape[2]))
    assert p.dtype == s.dtype == torch.float32
    rp, rs = MO.psnr_ssim(x.float().cpu().numpy(), y.float().cpu().numpy(), value_range)
    bp, bs = ssim_psnr_bounds(x, y, value_range, torch.from_numpy(rp).cuda(), torch.from_numpy(rs).cuda())
    assert np.all(bp <= PSNR_CAP) and np.all(bs <= SSIM_CAP), (bp.max(), bs.max())
    ep, es = np.abs(p.cpu().numpy() - rp), np.abs(s.cpu().numpy() - rs)
    print(f"psnr_ssim {shape} {dtype} {value_range}: psnr err/bound {(ep / bp).max():.3f}, ssim err/bound "
          f"{(es / bs).max():.3f} (ssim bound {bs.max():.2e})")
    assert np.all(ep <= bp), (ep.max(), bp.min())
    assert np.all(es <= bs), (es.max(), bs.min())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(3, 1, 11, 11), (2, 3, 40, 75), (2, 3, 4, 67, 129)])
def test_identical_inputs_are_exact(shape, dtype):
    import ops

    x, _ = make_inputs(shape, dtype, (0.0, 1.0), seed=1)
    p, s = ops.psnr_ssim(x, x.clone())
    assert torch.all(torch.isposinf(p)), p
    assert torch.all(s == 1.0), s


def test_bad_range_inputs_are_clamped_on_load():
    """Values past either end of the range score as the range's ends, exactly."""
    import ops

    x, y = make_inputs((2, 3, 3, 40, 50), torch.float32, (-1.0, 1.0), seed=3)
    x = x * 3
    p, s = ops.psnr_ssim(x, y, value_range=(-1, 1))
    pc, sc = ops.psnr_ssim(x.clamp(-1, 1), y.clamp(-1, 1), value_range=(-1, 1))
    check_bits("psnr", p, pc)
    check_bits("ssim", s, sc)


# ---------------------------------------------------------------------------------------------------- memory safety
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(2, 3, 11, 11), (1, 3, 5, 43, 75), (3, 1, 2, 40, 33)])
def test_memory_safety_and_determinism(shape, dtype):
    """Inputs inside guard bands of NaN, +big or -big (all three must give the same bits: an over-read that reached the
    result would change it); outputs inside sentinel-filled guard bands: every item is written, nothing else is."""
    import native
    import ops

    x0, y0 = make_inputs(shape, dtype, (0.0, 1.0), seed=7)
    B, C = shape[:2]
    T = shape[2] if len(shape) == 5 else 1
    H, W = shape[-2:]
    n = x0.numel()
    tiles = -(-(H - 10) // ops.METRICS_TILE) * -(-(W - 10) // ops.METRICS_TILE)
    results = []
    for poison in (float("nan"), 1e30, -1e30):
        gx, gy = Guarded(n, dtype, poison="nan"), Guarded(n, dtype, poison="nan")
        gx.buf.fill_(poison)
        gy.buf.fill_(-poison if poison == poison else poison)
        gx.body.copy_(x0.reshape(-1))
        gy.body.copy_(y0.reshape(-1))
        for _ in range(2):  # the rerun must give the same bits
            gp, gs = Guarded(B * T, torch.float32), Guarded(B * T, torch.float32)
            work = Guarded(2 * B * T * C * tiles, torch.float32)
            native.check(native.load().vqb_psnr_ssim(gx.ptr(), gy.ptr(), int(dtype == torch.bfloat16), B, C, T, H, W,
                                                     0.0, 1.0, gp.ptr(), gs.ptr(), work.ptr(), work.n,
                                                     torch.cuda.current_stream().cuda_stream), "psnr_ssim")
            torch.cuda.synchronize()
            everything = torch.arange(B * T, device="cuda")
            check_stores(gp, everything, "psnr")
            check_stores(gs, everything, "ssim")
            check_stores(work, torch.arange(work.n, device="cuda"), "work")
            assert not torch.isnan(gp.body).any() and not torch.isnan(gs.body).any()
            results.append((gp.body.clone(), gs.body.clone()))
    for p, s in results[1:]:
        check_bits("psnr", p, results[0][0])
        check_bits("ssim", s, results[0][1])
    p, s = ops.psnr_ssim(x0, y0)
    check_bits("psnr vs ops", p.reshape(-1), results[0][0])
    check_bits("ssim vs ops", s.reshape(-1), results[0][1])


def test_noncontiguous_and_mixed_device_inputs_are_refused():
    import native
    import ops

    x = torch.rand(1, 3, 20, 20, device="cuda")
    n0 = native.launch_count()
    with pytest.raises(ValueError, match="contiguous"):
        ops.psnr_ssim(x.transpose(2, 3), x.transpose(2, 3))
    with pytest.raises(RuntimeError):
        ops.psnr_ssim(x, x.cpu())
    with pytest.raises(RuntimeError, match="not differentiable"):
        ops.psnr_ssim(x.requires_grad_(True), x.detach())
    assert native.launch_count() == n0


def test_large_clip_batch_reruns_bit_identically():
    import ops

    x, y = make_inputs((2, 3, 48, 256, 256), torch.float32, (-1.0, 1.0), seed=11)
    a = ops.psnr_ssim(x, y, value_range=(-1, 1))
    b = ops.psnr_ssim(x, y, value_range=(-1, 1))
    check_bits("psnr", a[0], b[0])
    check_bits("ssim", a[1], b[1])


# ---------------------------------------------------------------------------------------------------- peer
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_agrees_with_fp64_conv2d_peer(dtype):
    import ops

    shape = (2, 3, 48, 256, 256)
    x, y = make_inputs(shape, dtype, (-1.0, 1.0), seed=13)
    p, s = ops.psnr_ssim(x, y, value_range=(-1, 1))
    rp, rs = MO.psnr_ssim_torch(x, y, (-1, 1))
    bp, bs = ssim_psnr_bounds(x, y, (-1, 1), rp, rs)
    assert p.shape == s.shape == (2, 48)
    ep, es = (p.double() - rp).abs().cpu().numpy(), (s.double() - rs).abs().cpu().numpy()
    print(f"peer {dtype}: psnr err/bound {(ep / bp).max():.3f}, ssim err/bound {(es / bs).max():.3f}")
    assert np.all(bp <= PSNR_CAP) and np.all(bs <= SSIM_CAP)
    assert np.all(ep <= bp) and np.all(es <= bs)


# ---------------------------------------------------------------------------------------------------- evaluation
def _trainer(gan=True):
    import tae_trainer
    import utils

    vae, _ = make_tvae(SMALL, "tae_small", torch.float32)
    lp = utils.LPIPS()  # train mode, as train_video runs it
    lp.load_state_dict(seeded_sd(LP.lpips_state_dict_shapes(), "lpips"), strict=True)
    pd = None
    if gan:
        pd = utils.PatchDiscriminator()
        pd.load_state_dict(seeded_sd(LP.patchd_state_dict_shapes(), "patchd"), strict=True)
        pd = pd.cuda()
    return tae_trainer.VideoTrainer(vae, lp.cuda(), pd, disc_type="hinge", use_lecam=True, perceptual_frames=2,
                                    lr_vae=1e-4, lr_disc=1e-4)


def _clip(tag, B=1, T=4):
    return seeded.tensor(f"metrics/{tag}", (B, 3, T, 16, 16), 1.0, "uniform").cuda()


def test_evaluate_scores_the_posterior_mean():
    import ops

    tr = _trainer(gan=False)
    clips = [_clip("e0", B=2), _clip("e1")]
    ev = tr.evaluate(clips)
    assert tr.lpips.training, "evaluate did not restore LPIPS's train mode"
    assert set(ev) == {"psnr", "ssim", "lpips", "psnr_frames", "ssim_frames", "lpips_frames"}
    with torch.no_grad():
        ps, ss, ls = [], [], []
        tr.lpips.eval()
        for c in clips:
            z = tr.vae.encoder(c)
            dec = tr.vae.decoder(z[:, :z.shape[1] // 2].contiguous())
            p, s = ops.psnr_ssim(dec, c, value_range=(-1, 1))
            ps.append(p)
            ss.append(s)
            ls.append(tr.lpips(dec.clamp(-1, 1), c).view(p.shape))
        tr.lpips.train()
    for k, ref in (("psnr", ps), ("ssim", ss)):
        ref = torch.cat(ref)
        assert ev[f"{k}_frames"].shape == (3, 4)
        check_bits(k, ev[f"{k}_frames"], ref)
        assert ev[k] == float(ref.double().mean())
    # LPIPS sums its spatial means with fp32 atomics: equal to a few ulps, not bit for bit
    ref = torch.cat(ls)
    assert ev["lpips_frames"].shape == (3, 4)
    torch.testing.assert_close(ev["lpips_frames"], ref, rtol=1e-5, atol=0)
    assert abs(ev["lpips"] - float(ref.double().mean())) <= 1e-5 * abs(ev["lpips"])
    assert math.isfinite(ev["psnr"]) and 0 < ev["ssim"] < 1 and ev["lpips"] > 0


def _trainer_state(tr):
    """Every piece of state a step reads: weights and buffers, the TVAE's packed bf16 operands, module modes, AdamW
    parameters and moments, LeCam anchors, and the CPU and CUDA RNG states."""
    import ops

    out = {"rng_cpu": torch.get_rng_state(), "rng_cuda": torch.cuda.get_rng_state()}
    for name, m in (("vae", tr.vae), ("disc", tr.disc), ("lpips", tr.lpips)):
        for k, v in m.state_dict().items():
            out[f"{name}.{k}"] = v.detach().clone()
        out[f"{name}.modes"] = torch.tensor([mm.training for mm in m.modules()])
        for mname, mm in m.named_modules():
            cache = getattr(mm, "_packed", None)
            if isinstance(cache, ops.PackedCache):
                for key, ent in cache._store.items():
                    out[f"{name}.{mname}.packed.{key}"] = ent.out.clone()
    for name, opt in (("G", tr.optimizer_G), ("D", tr.optimizer_D)):
        out[f"opt{name}.params"] = opt.store.params.detach().clone()
        out[f"opt{name}.exp_avg"] = opt.exp_avg.detach().clone()
        out[f"opt{name}.exp_avg_sq"] = opt.exp_avg_sq.detach().clone()
    out["anchors"] = torch.stack([tr.lecam_anchor_real_logits, tr.lecam_anchor_fake_logits]).clone()
    return out


def test_evaluate_between_steps_leaves_no_trace():
    """evaluate between two steps leaves every piece of state the next step reads bit-identical (weights, packed bf16
    operands, AdamW moments, anchors, module modes, RNG states). The step itself is not bit-reproducible (GroupNorm
    statistics and LPIPS means are summed with fp32 atomics), so the end state of the trainer that evaluated is compared
    with two that did not: bit for bit where those two agree bit for bit (RNG states, modes, frozen LPIPS), and within
    a wide multiple of their own rerun spread elsewhere."""
    finals = []
    for with_eval in (False, False, True):
        torch.manual_seed(5)
        torch.cuda.manual_seed(5)
        tr = _trainer()
        tr.step(_clip("s0"))
        if with_eval:
            before = _trainer_state(tr)
            assert any(".packed." in k for k in before), "no packed operand was compared"
            tr.evaluate([_clip("e0", B=2)])
            after = _trainer_state(tr)
            assert before.keys() <= after.keys()  # a forward at a new shape may add a cache entry, never change one
            for k in before:
                check_bits(f"evaluate changed {k}", after[k], before[k])
        out = tr.step(_clip("s1"))
        st = {k: v for k, v in _trainer_state(tr).items() if ".packed." not in k}  # packed: weights at the end
        st["recon"] = out["reconstructed"].clone()
        finals.append(st)
    plain, plain2, evald = finals
    assert plain.keys() == plain2.keys() == evald.keys()
    assert any(k.startswith("optG.") for k in plain), "no optimizer state was compared"
    for k in plain:
        if torch.equal(plain[k], plain2[k]):
            check_bits(k, evald[k], plain[k])
        else:
            spread = (plain2[k].double() - plain[k].double()).norm()
            diff = (evald[k].double() - plain[k].double()).norm()
            # AdamW amplifies one-ulp gradient differences where the second moment is small: allow for the tail of
            # that spread, while an extra optimizer step or a perturbed weight would still be far outside it
            assert diff <= 100 * spread, (k, diff.item(), spread.item())


TOY = ["--vae_ch", "32", "--vae_ch_mult", "1,8", "--vae_num_res_blocks", "1", "--vae_z_channels", "4",
       "--clip_frames", "4", "--resolution", "32", "--batch_size", "1"]


def test_cli_logs_held_out_scores(tmp_path):
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR",
                                                            "MASTER_PORT")}
    env["VQB_OFFLINE"] = "1"
    p = subprocess.run([sys.executable, os.path.join(PKG, "tae_trainer.py")] + TOY +
                       ["--eval_clips", "2", "--max_steps", "2", "--evaluate_every_n_steps", "1", "--run_name", "ev"],
                       cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    log = p.stderr
    for key in ("eval_psnr", "eval_ssim", "eval_lpips"):
        assert log.count(key) == 2, (key, log)
    assert sorted(os.listdir(tmp_path / "ckpt" / "ev")) == ["tvae_step_1.pt", "tvae_step_2.pt"]
