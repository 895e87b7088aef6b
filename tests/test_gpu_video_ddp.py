"""GPU (-m gpu): data-parallel training of the video autoencoder (tae_trainer.VideoTrainer under a process group).

Each multi-rank case spawns two worker processes. With gloo both share cuda:0 (gloo stages CUDA tensors through the
host; NCCL refuses two ranks on one device); the NCCL cases run one rank per GPU and need two GPUs. Models are the
tae_small configuration (one Down/Up level, heads of 32) on 4×32² clips. Cases:
  a. the constructor broadcasts rank 0's TVAE, discriminator and LPIPS, and no bf16 operand packed from a rank's own
     weights by an earlier forward survives (a no-grad encoder forward is deterministic, DESIGN.md §3.7);
  b. the TVAE gradient after the all-reduce is the rank mean of the local gradients, to one fp32 rounding, and each
     local gradient is the gradient of a world-size-1 step on that rank's clip, frames and noise;
  c. the same for the discriminator's gradient, and the LeCam anchors are fed by rank-averaged logits;
  d. with the full loss stack, weights, AdamW moments and anchors agree bit for bit on every rank after every step;
  e. without a process group the step issues no collective;
  g. the torchrun entry point runs in one process, saves a checkpoint tae.TVAE loads, and --load_path resumes it.
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

from helpers import cosine, seeded_sd
from oracle import lpips_oracle as LP
from oracle import seeded
from test_gpu_tae import SMALL, make_tvae

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "vqgan-training_b200")
CLIP = (1, 3, 4, 32, 32)
CASES = ("broadcast", "tvae_grad", "disc_grad", "full_stack")


# ------------------------------------------------------------------------------------------------ worker side
def _digest(tensors):
    """sha256 over the bytes of `tensors`: equal digests = bitwise-equal tensors."""
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def _state(m):
    return list(m.parameters()) + list(m.buffers())


def _clip(rank, i=0):
    return seeded.tensor(f"video_ddp/x{rank}_{i}", CLIP, 1.0, "uniform").bfloat16().float().cuda()


def _trainer(lpips=False, gan=False, recompute=False):
    """VideoTrainer on the seeded tae_small weights (the same on every rank), 2 of the clip's 4 frames per step."""
    import tae_trainer
    import utils

    vae, _ = make_tvae(SMALL, "tae_small", torch.float32)
    lp = pd = None
    if lpips:
        lp = utils.LPIPS()  # train mode: per-rank dropout draws, as train_video runs it
        lp.load_state_dict(seeded_sd(LP.lpips_state_dict_shapes(), "lpips"), strict=True)
        lp = lp.cuda()
    if gan:
        pd = utils.PatchDiscriminator()
        pd.load_state_dict(seeded_sd(LP.patchd_state_dict_shapes(), "patchd"), strict=True)
        pd = pd.cuda()
    return tae_trainer.VideoTrainer(vae, lp, pd, disc_type="hinge", use_lecam=True, perceptual_frames=2, lr_vae=1e-4,
                                    lr_disc=1e-4, recompute=recompute)


def _snoop(wrapper, store, log):
    """Wraps wrapper.allreduce_grads: log the flat gradient buffer before and after the all-reduce."""
    reduce = wrapper.allreduce_grads

    def snooped():
        store.collect()  # every gradient in its slot (the all-reduce does the same first)
        log.append(store.grads.detach().clone())
        reduce()
        log.append(store.grads.detach().clone())

    wrapper.allreduce_grads = snooped


def _layout(store, module):
    names = {p: n for n, p in module.named_parameters()}
    return [(names[p], o, p.numel()) for p, o in zip(store.plist, store.offsets)]


def _case_broadcast(rank, out):
    import tae
    import tae_trainer
    import utils

    torch.manual_seed(100 + rank)  # every rank initialises its own, different weights
    vae = tae.TVAE(**SMALL.kwargs()).cuda()
    lp = utils.LPIPS().eval().cuda()
    pd = utils.PatchDiscriminator().cuda()
    x = _clip(0)
    with torch.no_grad():  # every conv of the TVAE, LPIPS and D packs its bf16 operand from this rank's weights
        vae(x)
        lp(x, x)
        pd(x)
    mods = {"tvae": vae, "disc": pd, "lpips": lp}
    res = {"before": {k: _digest(_state(m)) for k, m in mods.items()}}
    tae_trainer.VideoTrainer(vae, lp, pd, disc_type="hinge", use_lecam=True, lr_vae=1e-4, lr_disc=1e-4)
    res["after"] = {k: _digest(_state(m)) for k, m in mods.items()}
    with torch.no_grad():
        res["encoder"] = _digest([vae.encoder(x)])
        res["disc_out"] = _digest([pd(x)])
    return res


def _case_tvae_grad(rank, out):
    """MSE + z loss (lpips=None, no D): no GradNorm on the gradient path, so the all-reduce is the only coupling."""
    x = _clip(rank)
    tr = _trainer()
    log = []
    _snoop(tr._vae_dp, tr.optimizer_G.store, log)
    torch.manual_seed(20 + rank)  # seeds whose frame draws differ between the ranks
    tr.step(x)
    sel = tr.last_frames.clone()
    layout = _layout(tr.optimizer_G.store, tr.vae)
    dist.barrier()
    dist.destroy_process_group()
    refs = []  # world size 1, twice (the run-to-run noise of the GroupNorm statistics' atomics)
    for _ in range(2):
        t1 = _trainer()
        torch.manual_seed(20 + rank)  # the same frames (CPU generator) and ε (CUDA generator)
        t1.step(x)
        assert torch.equal(t1.last_frames, sel)
        refs.append(t1.optimizer_G.store.grads.detach().clone())
    torch.save({"local": log[0].cpu(), "reduced": log[1].cpu(), "ref": [r.cpu() for r in refs], "layout": layout,
                "frames": sel}, os.path.join(out, f"tvae_grad_{rank}.pt"))
    return {}


def _case_disc_grad(rank, out):
    import tae_trainer

    x = _clip(rank)
    tr = _trainer(gan=True)
    log, local_logits = [], []
    _snoop(tr._disc_dp, tr.optimizer_D.store, log)
    loss = tae_trainer.gan_disc_loss

    def recorded(real, fake, disc_type):
        r = loss(real, fake, disc_type)
        local_logits.append((float(r[1]), float(r[2])))
        return r

    tae_trainer.gan_disc_loss = recorded
    torch.manual_seed(40 + rank)
    out_ = tr.step(x)
    torch.save({"local": log[0].cpu(), "reduced": log[1].cpu()}, os.path.join(out, f"disc_grad_{rank}.pt"))
    return {"anchors": [float(tr.lecam_anchor_real_logits), float(tr.lecam_anchor_fake_logits)],
            "local_logits": local_logits[0], "frames": tr.last_frames.tolist(),
            "finite": bool(torch.isfinite(out_["overall_vae_loss"]))}


def _case_full_stack(rank, out):
    tr = _trainer(lpips=True, gan=True, recompute=True)
    g, d = tr.optimizer_G, tr.optimizer_D
    w0 = [g.store.params.clone(), d.store.params.clone()]
    torch.manual_seed(30 + rank)
    steps = []
    for i in range(3):
        o = tr.step(_clip(rank, i))
        steps.append({
            "tvae": _digest([g.store.params]), "disc": _digest([d.store.params]),
            "tvae_moments": _digest([g.exp_avg, g.exp_avg_sq]), "disc_moments": _digest([d.exp_avg, d.exp_avg_sq]),
            "anchors": _digest([tr.lecam_anchor_real_logits, tr.lecam_anchor_fake_logits]),
            "frames": tr.last_frames.tolist(),
            "losses": [float(o[k]) for k in ("overall_vae_loss", "perceptual_loss", "d_loss", "g_gan_loss")]})
    moved = [not torch.equal(w0[0], g.store.params), not torch.equal(w0[1], d.store.params)]
    return {"steps": steps, "moved": moved}


def _worker(rank, world, port, backend, case, out, q):
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), VQB_OFFLINE="1")
    os.environ.pop("VQB_DDP_OVERLAP", None)
    try:
        dev = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        timeout = datetime.timedelta(seconds=300)  # a failed peer ends the other rank's collectives
        if backend == "nccl":
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev, timeout=timeout)
        else:
            dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timeout)
        res = globals()[f"_case_{case}"](rank, out)
        torch.cuda.synchronize()
        if dist.is_initialized():
            dist.barrier()
            dist.destroy_process_group()
        q.put((rank, "ok", res))
    except BaseException:
        q.put((rank, "error", traceback.format_exc()))
        raise


# ------------------------------------------------------------------------------------------------ parent side
def _spawn(case, out, backend="gloo"):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30100 + (os.getpid() % 200) + 10 * CASES.index(case) + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, case, str(out), q)) for r in range(2)]
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
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [r[2] for r in sorted(res, key=lambda r: r[0])]


def _check_rank_mean(what, local0, local1, reduced0, reduced1):
    assert torch.equal(reduced0, reduced1), f"{what}: ranks hold different gradients after the all-reduce"
    assert not torch.equal(local0, local1), f"{what}: the ranks' local gradients are equal (the check is vacuous)"
    mean = (local0.double() + local1.double()) / 2
    err = (reduced0.double() - mean).abs()
    bound = 2.0 ** -23 * mean.abs() + 1e-38  # one fp32 rounding (one ulp) of the exact mean
    print(f"\n{what}: max |reduced - mean| {err.max().item():.3e}; local gradients rel diff "
          f"{((local0 - local1).norm() / local0.norm()).item():.3e}")
    assert bool((err <= bound).all()), f"{what}: the all-reduced gradient is not the rank mean"


def _check_against_world1(rank, local, ref_a, ref_b, layout):
    """The module-level rule of test_gpu_tae_train.py, with a second world-size-1 run as the peer: per tensor, cosine
    error within 1.5x the run-to-run cosine error plus 5e-3; worst norm-ratio error within 1.5x the run-to-run one
    plus 2 %."""
    keys, cos, pcos, ratio, pratio = [], [], [], [], []
    norms = {n: ref_a[o:o + k].norm().item() for n, o, k in layout}
    top = max(norms.values())
    for n, o, k in layout:
        if norms[n] <= 1e-3 * top:  # mathematically-zero gradients carry only noise
            continue
        a, r, b = local[o:o + k], ref_a[o:o + k], ref_b[o:o + k]
        keys.append(n)
        cos.append(cosine(a, r))
        pcos.append(cosine(b, r))
        ratio.append(a.norm().item() / norms[n])
        pratio.append(b.norm().item() / norms[n])
    cos, pcos, ratio, pratio = map(np.array, (cos, pcos, ratio, pratio))
    print(f"\nrank {rank} local vs world-size-1 over {len(keys)} tensors: cosine min {cos.min():.7f} (run to run "
          f"{pcos.min():.7f}); norm ratio [{ratio.min():.6f}, {ratio.max():.6f}]")
    bad = [(k, c, pc) for k, c, pc in zip(keys, cos, pcos) if 1 - c > 1.5 * (1 - pc) + 5e-3]
    assert not bad, bad
    assert np.abs(ratio - 1).max() <= 1.5 * np.abs(pratio - 1).max() + 0.02


def _tvae_grad(tmp_path, backend):
    _spawn("tvae_grad", tmp_path, backend)
    r0, r1 = (torch.load(tmp_path / f"tvae_grad_{r}.pt") for r in range(2))
    assert not torch.equal(r0["frames"], r1["frames"]), "the ranks drew the same frames"
    _check_rank_mean("TVAE", r0["local"], r1["local"], r0["reduced"], r1["reduced"])
    for rank, r in enumerate((r0, r1)):
        _check_against_world1(rank, r["local"], r["ref"][0], r["ref"][1], r["layout"])


def _full_stack(tmp_path, backend):
    s0, s1 = _spawn("full_stack", tmp_path, backend)
    for i, (a, b) in enumerate(zip(s0["steps"], s1["steps"])):
        for k in ("tvae", "disc", "tvae_moments", "disc_moments", "anchors"):
            assert a[k] == b[k], f"step {i}: {k} differ between the ranks"
        assert np.isfinite(a["losses"] + b["losses"]).all(), (a["losses"], b["losses"])
    assert any(a["frames"] != b["frames"] for a, b in zip(s0["steps"], s1["steps"])), "the ranks drew the same frames"
    assert s0["moved"] == s1["moved"] == [True, True], "the weights did not move"


def test_constructor_broadcasts_rank0_state_and_repacks(tmp_path):
    r0, r1 = _spawn("broadcast", tmp_path)
    for k in ("tvae", "disc", "lpips"):
        assert r0["before"][k] != r1["before"][k], f"{k}: the ranks started equal (the check is vacuous)"
        assert r0["after"][k] == r1["after"][k] == r0["before"][k], f"{k}: rank 1 does not hold rank 0's state"
    assert r0["encoder"] == r1["encoder"], "a bf16 operand packed from rank 1's own weights survived the broadcast"
    assert r0["disc_out"] == r1["disc_out"]


def test_tvae_gradient_is_the_rank_mean_of_world1_gradients(tmp_path):
    _tvae_grad(tmp_path, "gloo")


def test_discriminator_gradient_and_lecam_anchors(tmp_path):
    r0, r1 = _spawn("disc_grad", tmp_path)
    g0, g1 = (torch.load(tmp_path / f"disc_grad_{r}.pt") for r in range(2))
    _check_rank_mean("discriminator", g0["local"], g1["local"], g0["reduced"], g1["reduced"])
    assert r0["frames"] != r1["frames"] and r0["finite"] and r1["finite"]
    assert r0["anchors"] == r1["anchors"], "the LeCam anchors differ between the ranks"
    assert r0["local_logits"] != r1["local_logits"]
    # first step from zero anchors: anchor = 0.1 * the rank mean of the local mean logits
    for j in range(2):
        want = 0.1 * (r0["local_logits"][j] + r1["local_logits"][j]) / 2
        assert abs(r0["anchors"][j] - want) <= 1e-6 * abs(want) + 1e-9, (j, r0["anchors"][j], want)


def test_full_stack_ranks_stay_bitwise_consistent(tmp_path):
    _full_stack(tmp_path, "gloo")


def test_single_process_step_issues_no_collective(monkeypatch):
    assert not dist.is_initialized()

    def refuse(*a, **k):
        raise AssertionError("a collective was issued without a process group")

    for name in ("all_reduce", "broadcast", "all_gather", "reduce_scatter", "barrier"):
        monkeypatch.setattr(dist, name, refuse)
    tr = _trainer(lpips=True, gan=True)
    assert tr.vae is tr._vae_dp.module and tr.disc is tr._disc_dp.module
    torch.manual_seed(0)
    out = tr.step(_clip(0))
    assert all(bool(torch.isfinite(out[k])) for k in ("overall_vae_loss", "d_loss", "g_gan_loss"))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_nccl_tvae_gradient_is_the_rank_mean_of_world1_gradients(tmp_path):
    _tvae_grad(tmp_path, "nccl")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_nccl_full_stack_ranks_stay_bitwise_consistent(tmp_path):
    _full_stack(tmp_path, "nccl")


# ------------------------------------------------------------------------------------------------ entry point
TOY = ["--vae_ch", "32", "--vae_ch_mult", "1,8", "--vae_num_res_blocks", "1", "--vae_z_channels", "4",
       "--clip_frames", "4", "--resolution", "32", "--batch_size", "1"]


def _run_cli(args, cwd):
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR",
                                                            "MASTER_PORT")}
    env["VQB_OFFLINE"] = "1"
    p = subprocess.run([sys.executable, os.path.join(PKG, "tae_trainer.py")] + TOY + args, cwd=cwd, env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    return p.stderr


def test_cli_trains_saves_and_resumes_a_checkpoint(tmp_path):
    import tae

    log = _run_cli(["--do_ganloss", "--disc_type", "hinge", "--use_lecam", "True", "--perceptual_frames", "2",
                    "--recompute", "--max_steps", "3", "--evaluate_every_n_steps", "2", "--run_name", "toy"], tmp_path)
    assert "step 0" in log and "lecam_anchor_real_logits" in log and "ms_per_step" in log, log
    assert sorted(os.listdir(tmp_path / "ckpt" / "toy")) == ["tvae_step_2.pt"]
    ck = torch.load(tmp_path / "ckpt" / "toy" / "tvae_step_2.pt")
    m = tae.TVAE(**SMALL.kwargs() | {"resolution": 32})
    m.load_state_dict(ck, strict=True)
    torch.manual_seed(42)  # the initial weights of that run (--seed 42, rank 0)
    init = tae.TVAE(**SMALL.kwargs() | {"resolution": 32}).state_dict()
    assert any(not torch.equal(ck[k], init[k]) for k in init), "the weights did not move"
    # resume: the first step of the warm-up runs at learning rate 0, so the saved weights are the loaded ones
    _run_cli(["--no_lpips", "--load_path", str(tmp_path / "ckpt" / "toy" / "tvae_step_2.pt"), "--max_steps", "1",
              "--evaluate_every_n_steps", "1", "--run_name", "resumed"], tmp_path)
    ck2 = torch.load(tmp_path / "ckpt" / "resumed" / "tvae_step_1.pt")
    assert ck2.keys() == ck.keys() and all(torch.equal(ck2[k], ck[k]) for k in ck)
