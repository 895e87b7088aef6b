"""GPU (-m gpu): the weight EMA fused into the AdamW launch (vqb_adamw_ema_flat_dev, flat.FlatAdamW(ema_decay=...)) and
the averaged inference modules of the trainers (DESIGN.md section 7 row 26, oracle/ema_oracle.py).

  kernel bound       e' = e - r (e - p') against float64 over a ragged chunk layout (4 groups, chunks without a gradient,
                     zero pads), at n = 1, in the warm-up and past the cap; mutated references (the rate of n - 1 or
                     n + 1, the pre-update p, skipped inactive chunks, d in place of 1 - d) must be rejected
  no perturbation    p, m, v bit-identical to vqb_adamw_flat_dev on the same inputs
  Trainer            GAN + LeCam, 3 eager steps then graph replays: after every step the EMA buffer follows the fp64
                     recurrence over the parameters that step actually produced; ema_updates counts the steps; the
                     same native launches per replay with and without the EMA
  vae_ema            after further steps, its reconstructions equal those of a fresh module loaded with its state_dict
                     bit for bit (no stale bf16 operand), and differ from the live module's
  VideoTrainer       the recurrence check, eagerly, and the same inference check
  data parallel      two gloo ranks on one GPU hold bit-identical EMA buffers after 3 full-stack steps
  checkpoint         after load_vae_checkpoint the EMA equals the loaded weights

Training forwards are not bit-reproducible across runs (GroupNorm statistics are summed with fp32 atomics), so every
trajectory check compares quantities of one run only.
"""
import ctypes
import datetime
import hashlib
import os
import random
import sys
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ema_oracle
from test_gpu_kernel_bounds import DEV, K, Guarded, check, check_stores, lib, ok, rejects, stream  # noqa: F401
from test_gpu_loss_optim_bounds import GRAD_SCALE, adamw_groups, adamw_ref, nan_guarded

pytestmark = pytest.mark.gpu

u = 2.0 ** -24
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "vqgan-training_b200")
DECAY = 0.999


# ---------------------------------------------------------------------------------------------------- kernel
def ragged_layout(gen, ntensors=900):
    """A FlatParams-like layout: tensors of ragged sizes, each padded to whole 1024-element chunks, each in one of 4
    groups or (no gradient this step) 255. -> (chunk groups [nchunks] uint8, pad mask [n] bool)."""
    sizes = torch.randint(1, 5000, (ntensors,), generator=gen)
    sizes[:5] = torch.tensor([1, 1023, 1024, 1025, 4096])
    groups = torch.randint(0, 5, (ntensors,), generator=gen)
    groups[groups == 4] = 255
    cg, pad = [], []
    for s, g in zip(sizes.tolist(), groups.tolist()):
        nc = -(-s // 1024)
        cg += [g] * nc
        m = torch.zeros(nc * 1024, dtype=torch.bool)
        m[s:] = True
        pad.append(m)
    return torch.tensor(cg, dtype=torch.uint8), torch.cat(pad)


def ema_bound(e, p1, e1, r):
    """e' = fl(e - r fl(e - p')): the difference rounds once (u |e - p'|, scaled by r), the update once more, fused or
    not (u |e'|, and u r |e - p'| for a separately rounded product): 2 u r |e - p'| + u |e'| to first order. Taken as
    3 u r |e - p'| + 2 u |e'| for the second-order terms."""
    return 3 * u * r * (e - p1).abs() + 2 * u * e1.abs()


@pytest.mark.parametrize("n", [1, 100, 20000])  # the first update, the warm-up (d = 101/110), past the cap
def test_adamw_ema_kernel_bounds(n):
    L = K.L
    gen = torch.Generator().manual_seed(n)
    cg, pad = ragged_layout(gen)
    nchunk, numel = cg.numel(), cg.numel() * 1024
    assert nchunk > 16 * 132 and all(int((cg == k).sum()) > 50 for k in (0, 1, 2, 3, 255)) and pad.sum() > 10 ** 5
    cg, pad = cg.to(DEV), pad.to(DEV)
    dg = torch.Generator(device=DEV).manual_seed(n)
    p0 = torch.randn(numel, device=DEV, generator=dg)
    g0 = torch.randn(numel, device=DEV, generator=dg) * 10 ** (torch.rand(numel, device=DEV, generator=dg) * 4 - 3)
    m0 = torch.randn(numel, device=DEV, generator=dg) * 0.01
    v0 = torch.rand(numel, device=DEV, generator=dg) * 1e-3
    e0 = p0 + 0.05 * torch.randn(numel, device=DEV, generator=dg)  # an average near the weights
    for x in (p0, g0, m0, v0, e0):
        x[pad] = 0.0  # the store's pads
    cgb = torch.zeros(nchunk + 8192, dtype=torch.uint8, device=DEV)  # group 0 around the table: an over-read moves guards
    cgb[4096:4096 + nchunk] = cg
    Gg = nan_guarded(g0)
    rec_host = (ctypes.c_float * 28)()
    ok(L.vqb_adamw_fill_record(4, adamw_groups(7), rec_host), "adamw_fill_record")
    rec32 = torch.tensor(list(rec_host), dtype=torch.float32, device=DEV)
    REC = nan_guarded(rec32)
    r = float(ema_oracle.rate_at(n, DECAY))
    RATE = nan_guarded(torch.tensor([r], device=DEV))

    def run(ema):
        P, M, V, E = (Guarded(numel, torch.float32) for _ in range(4))
        for B, x in ((P, p0), (M, m0), (V, v0), (E, e0)):
            B.body.copy_(x)
        if ema:
            rc = L.vqb_adamw_ema_flat_dev(P.ptr(), Gg.ptr(), M.ptr(), V.ptr(), E.ptr(), cgb.data_ptr() + 4096, nchunk,
                                          REC.ptr(), RATE.ptr(), GRAD_SCALE, stream())
        else:
            rc = L.vqb_adamw_flat_dev(P.ptr(), Gg.ptr(), M.ptr(), V.ptr(), cgb.data_ptr() + 4096, nchunk, REC.ptr(),
                                      GRAD_SCALE, stream())
        ok(rc, "adamw_ema_flat_dev" if ema else "adamw_flat_dev")
        torch.cuda.synchronize()
        for B, nm in ((P, "p"), (M, "m"), (V, "v"), (E, "ema")):
            check_stores(B, torch.arange(numel, device=DEV), f"{nm} stores")
        return P, M, V, E

    P, M, V, E = run(True)
    name = f"adamw_ema n={n} r={r:.6g} chunks={nchunk}"
    # no perturbation: the optimizer's outputs are those of the kernel without the average, bit for bit
    P0, M0, V0, E0 = run(False)
    for a, b, nm in ((P, P0, "p"), (M, M0, "m"), (V, V0, "v")):
        assert torch.equal(a.bits(), b.bits()), f"{name}: {nm} differs from vqb_adamw_flat_dev"
    assert torch.equal(E0.body.view(torch.int32), e0.view(torch.int32))  # (the plain kernel leaves ema alone)
    # the AdamW half is still within the bounds of test_gpu_loss_optim_bounds.py
    (pr, _, _), (bp, _, _) = adamw_ref(p0, g0, m0, v0, cg, rec32.double().view(7, 4), float(np.float32(GRAD_SCALE)))
    check(name + " p", P.body, pr, bp)

    p1 = P.body.double()
    e = e0.double()
    want = ema_oracle.update(e.cpu().numpy(), p1.cpu().numpy(), r)
    want = torch.from_numpy(want).to(DEV)
    bound = ema_bound(e, p1, want, r)
    check(name + " ema", E.body, want, bound)
    assert (E.body[pad] == 0).all() and (E.body.view(torch.int32)[pad] == 0).all(), f"{name}: a pad moved"
    inactive = (cg == 255).repeat_interleave(1024) & ~pad
    assert not torch.equal(E.body[inactive], e0[inactive]), f"{name}: chunks without a gradient were not averaged"
    again = run(True)
    assert torch.equal(E.bits(), again[3].bits()), f"{name}: two runs differ"

    # the bound bites
    got = E.body
    for m in (n - 1, n + 1):
        if m >= 1 and ema_oracle.decay_at(m, DECAY) != ema_oracle.decay_at(n, DECAY):  # (equal past the cap)
            rm = float(ema_oracle.rate_at(m, DECAY))
            rejects(f"{name}: the rate of n={m}", got, e - rm * (e - p1), bound)
    rejects(name + ": the pre-update p", got, e - r * (e - p0.double()), bound)
    rejects(name + ": inactive chunks skipped", got, torch.where(inactive, e, want), bound)
    d = float(np.float32(1.0 - r))
    rejects(name + ": d in place of 1 - d", got, e - d * (e - p1), bound)


# ---------------------------------------------------------------------------------------------------- trainers
class Recurrence:
    """The fp64 EMA recurrence over the parameter snapshots of one run, with its accumulated error bound: the error of
    the previous average decays by d_n, and each update adds ema_bound."""

    def __init__(self, opt):
        self.opt, self.decay = opt, opt.ema_decay
        self.e = opt.ema.double()
        self.b = torch.zeros_like(self.e)
        self.n = opt.ema_updates
        assert torch.equal(opt.ema, opt.store.params), "the average does not start from the weights"

    def after_step(self, what):
        torch.cuda.synchronize()
        opt = self.opt
        self.n += 1
        assert opt.ema_updates == self.n, (what, opt.ema_updates, self.n)
        r = float(ema_oracle.rate_at(self.n, self.decay))
        p1 = opt.store.params.double()
        e1 = self.e - r * (self.e - p1)
        self.b = (1 - r) * self.b + ema_bound(self.e, p1, e1, r)
        self.e = e1
        return check(f"{what} n={self.n} r={r:.4g}", opt.ema, self.e, self.b)


def _image_trainer(ema_decay=None, graph=True, seed=42):
    import vae_trainer as vt

    return vt.Trainer("cuda:0", vae_resolution=64, vae_ch=32, vae_ch_mult="1,2", vae_num_res_blocks=1,
                      vae_z_channels=4, do_clamp=True, do_ganloss=True, disc_type="hinge", use_lecam=True,
                      max_steps=50, learning_rate_vae=2e-2, lpips_eval=True, cuda_graph=graph, seed=seed,
                      ema_decay=ema_decay)


def _fresh_vae():
    import ae

    return ae.VAE(resolution=64, in_channels=3, ch=32, out_ch=3, ch_mult=[1, 2], num_res_blocks=1, z_channels=4,
                  use_attn=False, decoder_also_perform_hr=False, use_wavelet=False).cuda()


def _batches():
    g = torch.Generator().manual_seed(9)
    return [(torch.rand(2, 3, 256, 256, generator=g) * 2 - 1).pin_memory() for _ in range(3)]


def test_trainer_ema_follows_the_recurrence_under_graph_replay():
    """Decay 0.4: the warm-up (2/11, 3/12, ...) reaches the cap at n = 5, inside the 12 steps."""
    batches = _batches()
    tr = _image_trainer(ema_decay=0.4)
    opt = tr.optimizer_G
    assert tr.optimizer_D.ema is None
    rec = Recurrence(opt)
    random.seed(123)
    x = batches[0].cuda()
    for i in range(8):
        tr.step(batches[i % 3])
        rec.after_step(f"Trainer step {i} ({'graph' if i >= tr.GRAPH_WARMUP_STEPS else 'eager'})")
    assert tr.graph_launches_per_step is not None and opt.ema_updates == 8 == opt.param_groups[0]["step"]

    # vae_ema: its packs are built now, go stale over the next steps and must be refreshed on the next use
    with torch.no_grad():
        tr.vae_ema(x)
    for i in range(8, 12):
        tr.step(batches[i % 3])
        rec.after_step(f"Trainer step {i} (graph)")
    with torch.no_grad():
        got = tr.vae_ema(x)[0]
        live = tr.vae.module(x)[0]
        fresh = _fresh_vae()
        fresh.load_state_dict(tr.vae_ema.state_dict(), strict=True)
        want = fresh(x)[0]
    torch.cuda.synchronize()
    print(f"  vae_ema vs fresh module: bit-identical={torch.equal(got, want)}; vs live: max |diff| "
          f"{(got - live).abs().max().item():.3g}", flush=True)
    assert torch.equal(got, want), "vae_ema ran on stale packed operands"
    assert not torch.equal(got, live), "the averaged weights reconstruct like the live ones"
    ev = tr.evaluate([batches[0]], ema=True)
    assert torch.isfinite(ev["raw_reconstructed"]).all()
    ev_live = tr.evaluate([batches[0]])
    assert not torch.equal(ev["raw_reconstructed"], ev_live["raw_reconstructed"])
    launches_ema = tr.graph_launches_per_step
    tr.release_graph()

    plain = _image_trainer()
    assert plain.vae_ema is None and plain.optimizer_G.ema is None
    random.seed(123)
    for i in range(4):
        plain.step(batches[i % 3])
    print(f"  native launches per replay: {launches_ema} with EMA, {plain.graph_launches_per_step} without",
          flush=True)
    assert plain.graph_launches_per_step == launches_ema
    plain.release_graph()


def test_checkpoint_load_restarts_the_average_on_the_loaded_weights():
    import vae_trainer as vt

    batches = _batches()
    src = _image_trainer(graph=False, seed=5)
    for i in range(2):
        src.step(batches[i])
    sd = {k: v.detach().clone() for k, v in src.vae.state_dict().items()}
    tr = _image_trainer(ema_decay=DECAY, graph=False)
    x = batches[0].cuda()
    with torch.no_grad():
        before = tr.vae_ema(x)[0]  # packs from the random init
    vt.load_vae_checkpoint(tr.vae, sd)
    opt = tr.optimizer_G
    assert opt.ema_updates == 0 and torch.equal(opt.ema, opt.store.params)
    esd = tr.vae_ema.state_dict()
    assert all(torch.equal(esd[k], sd["module." + k]) for k in esd)
    with torch.no_grad():
        got, live = tr.vae_ema(x)[0], tr.vae.module(x)[0]
    assert torch.equal(got, live) and not torch.equal(got, before)
    rec = Recurrence(opt)
    tr.step(batches[1])
    rec.after_step("Trainer step after load")


def _video_trainer(ema_decay=None, lpips=False):
    import tae_trainer
    import utils
    from helpers import seeded_sd
    from oracle import lpips_oracle as LP
    from test_gpu_tae import SMALL, make_tvae

    vae, _ = make_tvae(SMALL, "tae_small", torch.float32)
    pd = utils.PatchDiscriminator()
    pd.load_state_dict(seeded_sd(LP.patchd_state_dict_shapes(), "patchd"), strict=True)
    lp = None
    if lpips:
        lp = utils.LPIPS()
        lp.load_state_dict(seeded_sd(LP.lpips_state_dict_shapes(), "lpips"), strict=True)
        lp = lp.cuda()
    return tae_trainer.VideoTrainer(vae, lp, pd.cuda(), disc_type="hinge", use_lecam=True, perceptual_frames=2,
                                    lr_vae=1e-4, lr_disc=1e-4, ema_decay=ema_decay)


def _clip(rank, i=0):
    from oracle import seeded

    return seeded.tensor(f"video_ddp/x{rank}_{i}", (1, 3, 4, 32, 32), 1.0, "uniform").bfloat16().float().cuda()


def test_video_trainer_ema_follows_the_recurrence():
    import tae
    from test_gpu_tae import SMALL

    tr = _video_trainer(ema_decay=0.4)
    rec = Recurrence(tr.optimizer_G)
    torch.manual_seed(3)
    x = _clip(0)
    for i in range(6):
        tr.step(_clip(0, i % 2))
        rec.after_step(f"VideoTrainer step {i}")
        if i == 2:
            with torch.no_grad():
                tr.vae_ema.encoder(x)  # pack now; the next steps make these operands stale
    with torch.no_grad():
        def recon(m):
            z = m.encoder(x)
            return m.decoder(z[:, :z.shape[1] // 2])

        fresh = tae.TVAE(**SMALL.kwargs()).cuda()
        fresh.load_state_dict(tr.vae_ema.state_dict(), strict=True)
        got, want, live = recon(tr.vae_ema), recon(fresh), recon(tr.vae)
    assert torch.equal(got, want), "vae_ema ran on stale packed operands"
    assert not torch.equal(got, live)
    ev, ev_live = tr.evaluate([x], ema=True), tr.evaluate([x])
    assert np.isfinite(ev["psnr"]) and ev["psnr"] != ev_live["psnr"]
    assert tr.optimizer_D.ema is None


# ---------------------------------------------------------------------------------------------------- data parallel
def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def _worker(rank, world, port, out, q):
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), VQB_OFFLINE="1")
    os.environ.pop("VQB_DDP_OVERLAP", None)
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
        tr = _video_trainer(ema_decay=0.9, lpips=True)
        g = tr.optimizer_G
        res = {"init": _digest(g.ema), "steps": []}
        torch.manual_seed(30 + rank)
        for i in range(3):
            tr.step(_clip(rank, i))
            torch.cuda.synchronize()
            res["steps"].append({"ema": _digest(g.ema), "params": _digest(g.store.params), "n": g.ema_updates,
                                 "frames": tr.last_frames.tolist()})
        res["moved"] = not torch.equal(g.ema, g.store.params)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok", res))
    except BaseException:
        q.put((rank, "error", traceback.format_exc()))
        raise


def test_data_parallel_ranks_hold_identical_averages():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30700 + (os.getpid() % 200)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, "", q)) for r in range(2)]
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
    s0, s1 = (r[2] for r in sorted(res, key=lambda r: r[0]))
    assert s0["init"] == s1["init"], "the averages did not start from rank 0's broadcast weights"
    for i, (a, b) in enumerate(zip(s0["steps"], s1["steps"])):
        assert a["n"] == b["n"] == i + 1
        assert a["params"] == b["params"], f"step {i}: weights differ between the ranks"
        assert a["ema"] == b["ema"], f"step {i}: the EMA buffers differ between the ranks"
    assert any(a["frames"] != b["frames"] for a, b in zip(s0["steps"], s1["steps"])), "the ranks drew the same frames"
    assert s0["moved"] and s1["moved"]
