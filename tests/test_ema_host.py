"""CPU: the weight EMA of FlatAdamW and the trainers without a device. The schedule of oracle/ema_oracle.py and its
restatement in flat.py, the refusal of a bad decay before any allocation, launch or device work, the averaged
inference module over the EMA buffer (views, not copies; strict state_dict round trips into fresh ae.VAE / tae.TVAE
modules), the C ABI of vqb_adamw_ema_flat_dev and the --ema_decay flag of train_video."""
import ctypes
import inspect
import math
import os

import numpy as np
import pytest
import torch
from click.testing import CliRunner

from oracle import ema_oracle

EINVAL, ENODEVICE = -1, -2
BAD_DECAYS = (0.0, 1.0, -0.5, 1.5, math.nan, math.inf)
SMALL = dict(vae_resolution=32, vae_ch=32, vae_ch_mult="1,2", vae_num_res_blocks=1, vae_z_channels=4, max_steps=10)


# ---------------------------------------------------------------------------------------------------- schedule
def test_oracle_schedule_warms_up_then_caps():
    assert ema_oracle.decay_at(1, 0.999) == 2 / 11  # the first update
    assert ema_oracle.decay_at(2, 0.999) == 3 / 12
    assert ema_oracle.decay_at(1, 0.1) == 0.1       # a decay below 2/11 caps from the start
    # (1 + n) / (10 + n) reaches 0.999 at n = 8990: the warm-up hands over to the cap there
    assert ema_oracle.decay_at(8989, 0.999) < 0.999 and ema_oracle.decay_at(8991, 0.999) == 0.999
    assert ema_oracle.decay_at(10 ** 6, 0.999) == 0.999
    assert ema_oracle.rate_at(1, 0.999) == np.float32(9 / 11)
    with pytest.raises(ValueError):
        ema_oracle.decay_at(0, 0.999)  # n is incremented before use: there is no update 0


def test_oracle_recurrence_counts_updates_from_one():
    e0, p = np.array([1.0, -2.0, 0.0]), [np.array([0.0, 0.0, 0.0]), np.array([3.0, 1.0, 0.0])]
    e1, e2 = ema_oracle.recurrence(e0, p, 0.9)
    r1, r2 = float(np.float32(9 / 11)), float(np.float32(1 - 3 / 12))
    assert np.array_equal(e1, e0 - r1 * (e0 - p[0]))
    assert np.array_equal(e2, e1 - r2 * (e1 - p[1]))
    assert e2[2] == 0.0  # a zero pad stays zero
    # resuming the recurrence at n0 continues the count
    (e2b,) = ema_oracle.recurrence(e1, p[1:], 0.9, n0=1)
    assert np.array_equal(e2, e2b)


@pytest.mark.parametrize("decay", [0.5, 0.9, 0.999, 0.9999, 1e-3])
def test_flat_schedule_matches_the_oracle(decay):
    import flat

    for n in list(range(1, 200)) + [8989, 8990, 8991, 10 ** 5, 10 ** 7]:
        assert flat.ema_decay_at(n, decay) == ema_oracle.decay_at(n, decay)
        assert flat.ema_rate(n, decay) == float(ema_oracle.rate_at(n, decay)), n


@pytest.mark.parametrize("decay", BAD_DECAYS + ("x", None))
def test_bad_decays_are_refused(decay):
    import flat

    if decay is None:
        return  # None means "no EMA", not a bad value
    with pytest.raises(ValueError):
        flat.check_ema_decay(decay)
    if isinstance(decay, float):
        with pytest.raises(ValueError):
            ema_oracle.check_decay(decay)


def _count_allocs(monkeypatch):
    """Counts torch.zeros / empty / clone calls and refuses any native launch."""
    import native

    calls = []
    for name in ("zeros", "empty"):
        real = getattr(torch, name)
        monkeypatch.setattr(torch, name, lambda *a, _r=real, **k: (calls.append(1), _r(*a, **k))[1])
    monkeypatch.setattr(native, "load", lambda: pytest.fail("a native entry point was loaded"))
    return calls


@pytest.mark.parametrize("decay", BAD_DECAYS)
def test_bad_decay_fails_before_any_allocation(decay, monkeypatch):
    import flat
    import tae_trainer
    import vae_trainer

    p, lin = torch.nn.Parameter(torch.ones(3)), torch.nn.Linear(1, 1)
    calls = _count_allocs(monkeypatch)
    with pytest.raises(ValueError, match="ema_decay"):
        flat.FlatAdamW([{"params": [p], "lr": 1e-3}], ema_decay=decay)
    with pytest.raises(ValueError, match="ema_decay"):
        vae_trainer.Trainer("cuda", ema_decay=decay, **SMALL)  # refused before any module is built on a device
    with pytest.raises(ValueError, match="ema_decay"):
        tae_trainer.VideoTrainer(lin, None, lr_vae=1e-4, ema_decay=decay)
    assert calls == []
    assert p.data_ptr() and torch.equal(p.data, torch.ones(3))  # not re-homed


def test_no_decay_is_todays_optimizer():
    import flat

    p = torch.nn.Parameter(torch.randn(5, 7))
    opt = flat.FlatAdamW([{"params": [p], "lr": 1e-3}])
    assert opt.ema is None and opt.ema_decay is None and opt.ema_updates == 0
    with pytest.raises(RuntimeError):
        opt.reset_ema()
    with pytest.raises(RuntimeError):
        opt.averaged_copy(torch.nn.Linear(1, 1))
    for cls in ("Trainer",):
        import vae_trainer

        assert inspect.signature(getattr(vae_trainer, cls)).parameters["ema_decay"].default is None
    import tae_trainer

    assert inspect.signature(tae_trainer.VideoTrainer).parameters["ema_decay"].default is None


# ---------------------------------------------------------------------------------------------------- CPU storage
def test_flat_adamw_ema_buffer_and_reset():
    import flat

    torch.manual_seed(0)
    a, b = torch.nn.Parameter(torch.randn(3, 5)), torch.nn.Parameter(torch.randn(1500))
    opt = flat.FlatAdamW([{"params": [a], "lr": 1e-3}, {"params": [b], "lr": 1e-4}], ema_decay=0.999)
    st = opt.store
    assert opt.ema.shape == st.params.shape == (2048 + 1024,) and opt.ema.dtype == torch.float32
    assert opt.ema.data_ptr() != st.params.data_ptr()
    assert torch.equal(opt.ema, st.params) and opt.ema_updates == 0
    with torch.no_grad():
        a.add_(1.0)
    opt.ema_updates, g0 = 5, opt.ema_generation
    opt.reset_ema()
    assert torch.equal(opt.ema, st.params) and opt.ema_updates == 0 and opt.ema_generation > g0
    assert (opt.ema[15:1024] == 0).all() and (opt.ema[1024 + 1500:] == 0).all()  # pads


def _vae(**kw):
    import ae

    return ae.VAE(resolution=32, in_channels=3, ch=32, out_ch=3, ch_mult=[1, 2], num_res_blocks=1, z_channels=4,
                  use_attn=False, decoder_also_perform_hr=False, use_wavelet=False, **kw)


def _check_averaged(avg, live, opt, cls_factory):
    """avg's trainable parameters are views of opt.ema; its state_dict round-trips strictly into a fresh module."""
    ema = opt.ema
    lo, hi = ema.data_ptr(), ema.data_ptr() + 4 * ema.numel()
    trained = {id(p) for p in opt.store.plist}
    names = dict(live.named_parameters())
    nviews = 0
    for n, q in avg.named_parameters():
        p = names[n]
        assert q.shape == p.shape and not q.requires_grad, n
        if id(p) in trained:
            assert lo <= q.data_ptr() < hi and q.untyped_storage().data_ptr() == ema.untyped_storage().data_ptr(), n
            nviews += 1
        else:
            assert q.data_ptr() != p.data_ptr() and torch.equal(q, p), n
    assert nviews == len(opt.store.plist)
    for (n, q), (m, p) in zip(avg.named_buffers(), live.named_buffers()):
        assert n == m and q.data_ptr() != p.data_ptr() and torch.equal(q, p)
    for m in avg.modules():  # own pack caches
        if hasattr(m, "_packed"):
            assert m._packed is not dict(live.named_modules())[[k for k, v in avg.named_modules() if v is m][0]]._packed
    sd = avg.state_dict()
    assert list(sd) == list(live.state_dict())
    fresh = cls_factory()
    fresh.load_state_dict(sd, strict=True)
    assert all(torch.equal(fresh.state_dict()[k], sd[k]) for k in sd)
    # writes to the EMA buffer show through
    with torch.no_grad():
        ema.add_(0.25)
    k = next(n for n, p in live.named_parameters() if id(p) in trained)
    assert torch.equal(avg.state_dict()[k], live.state_dict()[k] + 0.25)
    with torch.no_grad():
        ema.sub_(0.25)


@pytest.mark.parametrize("use_vq", [False, True])
def test_trainer_on_cpu_keeps_an_averaged_vae(use_vq):
    import ae
    import vae_trainer as vt

    tr = vt.Trainer("cpu", ema_decay=0.999, use_vq=use_vq, vq_codebook_size=64, **SMALL)
    opt = tr.optimizer_G
    assert opt.ema_decay == 0.999 and opt.ema.numel() == opt.store.total
    assert tr.optimizer_D.ema is None  # the discriminator keeps no average
    live = tr.vae.module
    assert type(tr.vae_ema) is ae.VAE and tr.vae_ema is not live
    assert isinstance(tr.vae_ema.reg, ae.VectorQuantizer) == use_vq
    if use_vq:  # the codebook group is averaged too
        q = tr.vae_ema.reg.embedding.weight
        assert opt.ema.data_ptr() <= q.data_ptr() < opt.ema.data_ptr() + 4 * opt.ema.numel()

    def fresh():
        m = _vae()
        if use_vq:
            m.reg = ae.VectorQuantizer(64, 4, 0.25)
        return m

    _check_averaged(tr.vae_ema, live, opt, fresh)
    assert vt.Trainer("cpu", **SMALL).vae_ema is None


def test_checkpoint_load_restarts_the_average():
    import vae_trainer as vt

    tr = vt.Trainer("cpu", ema_decay=0.99, **SMALL)
    other = vt.Trainer("cpu", seed=7, **SMALL)
    sd = other.vae.state_dict()
    tr.optimizer_G.ema_updates = 3
    vt.load_vae_checkpoint(tr.vae, sd)
    assert tr.optimizer_G.ema_updates == 0
    esd = tr.vae_ema.state_dict()
    assert all(torch.equal(esd[k], sd["module." + k]) for k in esd)


def test_video_trainer_on_cpu_keeps_an_averaged_tvae():
    import tae
    import tae_trainer

    def fresh():
        torch.manual_seed(3)
        return tae.TVAE(resolution=16, in_channels=3, ch=32, out_ch=3, ch_mult=[1, 2], num_res_blocks=1, z_channels=4)

    vae = fresh()
    tr = tae_trainer.VideoTrainer(vae, None, lr_vae=1e-4, ema_decay=0.9)
    assert type(tr.vae_ema) is tae.TVAE
    _check_averaged(tr.vae_ema, vae, tr.optimizer_G, fresh)
    assert tae_trainer.VideoTrainer(fresh(), None, lr_vae=1e-4).vae_ema is None
    with pytest.raises(ValueError, match="EMA"):
        tae_trainer.VideoTrainer(fresh(), None, lr_vae=1e-4).evaluate([], ema=True)


# ---------------------------------------------------------------------------------------------------- C ABI
@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    L = native.load()
    L.vqb_last_error.restype = ctypes.c_char_p
    return L


def _expect(L, rc, code):
    name = "vqb_adamw_ema_flat_dev"
    err = L.vqb_last_error()
    assert rc == code, (rc, err)
    assert name.encode() in err, err
    if code == ENODEVICE:
        assert b"sm_90" in err, err


def test_adamw_ema_entry_point_validates_then_needs_a_device(lib):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16  # never dereferenced
    f = lib.vqb_adamw_ema_flat_dev
    # params, grads, exp_avg, exp_avg_sq, ema, chunk_group | record_dev, ema_rate_dev
    for k in range(8):
        args = [p] * 8
        args[k] = None
        _expect(lib, f(*args[:6], 3, *args[6:], 1.0, None), EINVAL)
    for k, off in ((0, 4), (1, 8), (2, 12), (3, 4), (4, 8)):  # one fp32 buffer off its 16-byte alignment
        args = [p] * 5
        args[k] = p + off
        _expect(lib, f(*args, p, 3, p, p, 1.0, None), EINVAL)
    _expect(lib, f(p, p, p, p, p, p, 3001, p, p, 0.37, None), ENODEVICE)
    _expect(lib, f(p, p, p, p, p, p, 1, p + 4, p + 4, 1.0, None), ENODEVICE)  # record and rate need no alignment


def test_header_declares_the_entry_point():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "vqb200.h")) as fh:
        assert "int vqb_adamw_ema_flat_dev(" in fh.read()


# ---------------------------------------------------------------------------------------------------- CLI
def _cli(monkeypatch):
    import tae_trainer

    seen = {}
    monkeypatch.setattr(tae_trainer, "_train_video", lambda *a, **k: seen.update(args=a, kw=k))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: pytest.fail("device work before the check"))
    monkeypatch.delenv("RANK", raising=False)
    return tae_trainer, seen


def test_ema_decay_reaches_the_training_loop_as_a_keyword(monkeypatch):
    import tae_trainer

    assert inspect.signature(tae_trainer._train_video).parameters["ema_decay"].default is None
    tae_trainer, seen = _cli(monkeypatch)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    res = CliRunner().invoke(tae_trainer.train_video, ["--ema_decay", "0.999"])
    assert res.exit_code == 0, res.output
    assert seen["kw"] == {"ema_decay": 0.999}
    default_args = seen["args"]
    res = CliRunner().invoke(tae_trainer.train_video, ["--ema_decay", "0.99", "--eval_clips", "2"])
    assert res.exit_code == 0, res.output
    assert seen["kw"] == {"ema_decay": 0.99, "eval_clips": 2} and seen["args"] == default_args
    res = CliRunner().invoke(tae_trainer.train_video, [])
    assert res.exit_code == 0, res.output
    assert seen["kw"] == {} and seen["args"] == default_args


@pytest.mark.parametrize("value", ["0", "1", "-0.1", "1.5", "nan", "inf"])
def test_bad_ema_decay_is_refused_before_device_work(monkeypatch, value):
    tae_trainer, seen = _cli(monkeypatch)
    res = CliRunner().invoke(tae_trainer.train_video, ["--ema_decay", value])
    assert res.exit_code == 2, res.output  # click.BadParameter
    assert "--ema_decay" in res.output and not seen


def test_train_ddp_gets_no_ema_flag():
    import vae_trainer

    assert not any(p.name == "ema_decay" for p in vae_trainer.train_ddp.params)
