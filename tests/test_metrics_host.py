"""CPU: the reconstruction metrics without a GPU. The float64 oracle (oracle/metrics_oracle.py) against closed forms,
cv2.PSNR and a brute-force window loop; ops.psnr_ssim refuses every bad call before anything launches; the C entry
point vqb_psnr_ssim returns VQB_EINVAL for bad arguments and VQB_ENODEVICE without a device; train_video refuses a
negative --eval_clips and passes a positive one through."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch
from click.testing import CliRunner

from oracle import metrics_oracle as MO

EINVAL, ENODEVICE = -1, -2


# ---------------------------------------------------------------------------------------------------- oracle
def _rand(shape, seed, lo=0.0, hi=1.0):
    return np.random.default_rng(seed).uniform(lo, hi, size=shape).astype(np.float32)


@pytest.mark.parametrize("shape", [(2, 3, 16, 20), (1, 1, 3, 11, 11), (2, 3, 2, 13, 17)])
def test_identical_inputs_give_inf_and_one(shape):
    x = _rand(shape, 0)
    p, s = MO.psnr_ssim(x, x.copy())
    assert p.shape == s.shape == ((shape[0],) if len(shape) == 4 else (shape[0], shape[2]))
    assert np.all(np.isposinf(p))
    np.testing.assert_allclose(s, 1.0, rtol=0, atol=1e-12)


@pytest.mark.parametrize("c1, c2", [(0.25, 0.625), (0.0, 1.0), (0.5, 0.5 + 2 ** -10), (0.875, 0.125)])
def test_constant_planes_have_the_closed_form(c1, c2):
    x = np.full((1, 3, 15, 19), c1, np.float32)
    y = np.full((1, 3, 15, 19), c2, np.float32)
    p, s = MO.psnr_ssim(x, y)
    # a constant window has no variance: only the luminance term of SSIM is left
    np.testing.assert_allclose(s, (2 * c1 * c2 + MO.C1) / (c1 ** 2 + c2 ** 2 + MO.C1), rtol=1e-12)
    np.testing.assert_allclose(p, -20 * math.log10(abs(c1 - c2)), rtol=1e-12)


@pytest.mark.parametrize("seed", [0, 1])
def test_psnr_agrees_with_cv2(seed):
    cv2 = pytest.importorskip("cv2")
    x, y = _rand((1, 3, 24, 31), seed), _rand((1, 3, 24, 31), seed + 10)
    ref = cv2.PSNR(np.transpose(x[0], (1, 2, 0)).astype(np.float64) * 255,
                   np.transpose(y[0], (1, 2, 0)).astype(np.float64) * 255, 255.0)
    p, _ = MO.psnr_ssim(x, y)
    assert abs(p[0] - ref) < 1e-9, (p[0], ref)


def test_valid_filter_equals_a_brute_force_loop():
    a = np.random.default_rng(3).standard_normal((2, 13, 17))
    w = MO.window()
    ref = np.zeros((2, 3, 7))
    for n in range(2):
        for p in range(3):
            for q in range(7):
                for i in range(11):
                    for j in range(11):
                        ref[n, p, q] += w[i, j] * a[n, p + i, q + j]
    np.testing.assert_allclose(MO.valid_filter(a), ref, rtol=0, atol=1e-13)


def test_window_is_symmetric_and_sums_to_one():
    g, w = MO.gaussian_1d(), MO.window()
    assert g.shape == (11,) and w.shape == (11, 11)
    np.testing.assert_array_equal(g, g[::-1])
    np.testing.assert_array_equal(w, w.T)
    assert abs(w.sum() - 1) < 1e-15 and abs(g.sum() - 1) < 1e-15
    assert int(np.argmax(g)) == 5
    np.testing.assert_allclose(g[4] / g[5], math.exp(-1 / (2 * 1.5 ** 2)), rtol=1e-15)


def test_out_of_range_values_are_clamped():
    u = MO.to_unit(np.array([-3.0, -1.0, 0.0, 0.5, 1.0, 7.0, np.nan, np.inf, -np.inf], np.float32), (-1, 1))
    np.testing.assert_array_equal(u, np.array([0, 0, 0.5, 0.75, 1, 1, 0, 1, 0], np.float32))
    assert u.dtype == np.float32
    x, y = _rand((2, 3, 2, 14, 12), 5, -3, 3), _rand((2, 3, 2, 14, 12), 6, -3, 3)
    for a, b in zip(MO.psnr_ssim(x, y, (-1, 1)), MO.psnr_ssim(np.clip(x, -1, 1), np.clip(y, -1, 1), (-1, 1))):
        np.testing.assert_array_equal(a, b)
    # (-1, 1) is the (0, 1) metric of (v + 1) / 2: exact in float32 for these inputs
    xs, ys = np.clip(x, -1, 1), np.clip(y, -1, 1)
    for a, b in zip(MO.psnr_ssim(xs, ys, (-1, 1)), MO.psnr_ssim((xs + 1) / 2, (ys + 1) / 2)):
        np.testing.assert_allclose(a, b, rtol=1e-6)


# ---------------------------------------------------------------------------------------------------- ops host checks
def _t(*shape, dtype=torch.float32, **kw):
    return torch.rand(*shape, dtype=dtype, **kw)


REFUSALS = [
    ("rank 3", lambda: (_t(3, 16, 16), _t(3, 16, 16)), {}, ValueError),
    ("rank 6", lambda: (_t(1, 1, 1, 1, 16, 16), _t(1, 1, 1, 1, 16, 16)), {}, ValueError),
    ("shape mismatch", lambda: (_t(1, 3, 16, 16), _t(1, 3, 16, 17)), {}, ValueError),
    ("dtype mismatch", lambda: (_t(1, 3, 16, 16), _t(1, 3, 16, 16, dtype=torch.bfloat16)), {}, ValueError),
    ("float16", lambda: (_t(1, 3, 16, 16, dtype=torch.float16),) * 2, {}, ValueError),
    ("float64", lambda: (_t(1, 3, 16, 16, dtype=torch.float64),) * 2, {}, ValueError),
    ("H < 11", lambda: (_t(1, 3, 10, 16), _t(1, 3, 10, 16)), {}, ValueError),
    ("W < 11", lambda: (_t(1, 3, 2, 16, 10), _t(1, 3, 2, 16, 10)), {}, ValueError),
    ("empty batch", lambda: (_t(0, 3, 16, 16), _t(0, 3, 16, 16)), {}, ValueError),
    ("empty clip", lambda: (_t(1, 3, 0, 16, 16), _t(1, 3, 0, 16, 16)), {}, ValueError),
    ("hi == lo", lambda: (_t(1, 3, 16, 16),) * 2, {"value_range": (1.0, 1.0)}, ValueError),
    ("hi < lo", lambda: (_t(1, 3, 16, 16),) * 2, {"value_range": (1.0, -1.0)}, ValueError),
    ("equal in float32", lambda: (_t(1, 3, 16, 16),) * 2, {"value_range": (1.0, 1.0 + 1e-9)}, ValueError),
    ("nan range", lambda: (_t(1, 3, 16, 16),) * 2, {"value_range": (0.0, float("nan"))}, ValueError),
    ("inf range", lambda: (_t(1, 3, 16, 16),) * 2, {"value_range": (-float("inf"), 1.0)}, ValueError),
    ("overflowing range", lambda: (_t(1, 3, 16, 16),) * 2, {"value_range": (0.0, 1e39)}, ValueError),
    ("not a pair", lambda: (_t(1, 3, 16, 16),) * 2, {"value_range": 1.0}, ValueError),
    ("cpu tensors", lambda: (_t(1, 3, 16, 16), _t(1, 3, 16, 16)), {}, RuntimeError),
    ("x requires grad", lambda: (_t(1, 3, 16, 16, requires_grad=True), _t(1, 3, 16, 16)), {}, RuntimeError),
    ("y requires grad", lambda: (_t(1, 3, 16, 16), _t(1, 3, 16, 16, requires_grad=True)), {}, RuntimeError),
]


@pytest.mark.parametrize("what, make, kw, exc", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_psnr_ssim_refuses_before_any_launch(what, make, kw, exc):
    import native
    import ops

    native.load()
    n0 = native.launch_count()
    x, y = make()
    with pytest.raises(exc):
        ops.psnr_ssim(x, y, **kw)
    assert native.launch_count() == n0


def test_inputs_that_require_grad_are_accepted_without_grad_mode():
    """Outside grad mode the value cannot become a loss: the call gets past the grad check (and stops at the device)."""
    import ops

    x = _t(1, 3, 16, 16, requires_grad=True)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA tensors only"):
        ops.psnr_ssim(x, x)


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


@pytest.fixture
def no_device():
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")


def _work(B, C, T, H, W):
    return 2 * B * T * C * (-(-(H - 10) // 32)) * (-(-(W - 10) // 32))


GOOD = dict(bf16=0, B=2, C=3, T=4, H=40, W=75, lo=-1.0, hi=1.0)
BAD_ABI = [
    ("x null", {}, "x"),
    ("y null", {}, "y"),
    ("psnr null", {}, "psnr"),
    ("ssim null", {}, "ssim"),
    ("work null", {}, "work"),
    ("bf16 = 2", {"bf16": 2}, None),
    ("B = 0", {"B": 0}, None),
    ("C = 0", {"C": 0}, None),
    ("T = 0", {"T": 0}, None),
    ("H = 10", {"H": 10}, None),
    ("W = 10", {"W": 10}, None),
    ("W < 0", {"W": -5}, None),
    ("hi == lo", {"lo": 0.5, "hi": 0.5}, None),
    ("hi < lo", {"lo": 1.0, "hi": 0.0}, None),
    ("nan", {"hi": float("nan")}, None),
    ("inf", {"lo": -float("inf")}, None),
    ("grid", {"B": 1 << 20, "T": 1 << 10, "H": 1000, "W": 1000}, None),
    ("work short", {"work": -1}, None),
]


def _call(L, args, null=None):
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    a = dict(GOOD)
    a.update({k: v for k, v in args.items() if k != "work"})
    work = _work(a["B"], a["C"], a["T"], max(a["H"], 11), max(a["W"], 11)) + args.get("work", 0)
    ptrs = {k: (None if k == null else p) for k in ("x", "y", "psnr", "ssim", "work")}
    return L.vqb_psnr_ssim(ptrs["x"], ptrs["y"], a["bf16"], a["B"], a["C"], a["T"], a["H"], a["W"], a["lo"], a["hi"],
                           ptrs["psnr"], ptrs["ssim"], ptrs["work"], work, None)


@pytest.mark.parametrize("what, args, null", BAD_ABI, ids=[b[0] for b in BAD_ABI])
def test_abi_rejects_bad_arguments(lib, what, args, null):
    rc = _call(lib, args, null)
    err = lib.vqb_last_error()
    assert rc == EINVAL, (what, rc, err)
    assert b"vqb_psnr_ssim" in err, err


@pytest.mark.parametrize("args", [{}, {"bf16": 1}, {"H": 11, "W": 11, "T": 1, "C": 1, "B": 1}])
def test_abi_without_device_is_enodevice(lib, no_device, args):
    rc = _call(lib, args)
    err = lib.vqb_last_error()
    assert rc == ENODEVICE, (rc, err)
    assert b"vqb_psnr_ssim" in err and b"sm_90" in err, err


# ---------------------------------------------------------------------------------------------------- CLI
def _guard_device(monkeypatch, tae_trainer):
    def device_work(*a, **k):
        raise AssertionError("device work before the arguments were checked")

    monkeypatch.setattr(torch.cuda, "is_available", device_work)
    monkeypatch.setattr(torch.cuda, "set_device", device_work)
    monkeypatch.setattr(tae_trainer, "_train_video", device_work)


def test_negative_eval_clips_is_refused_before_device_work(monkeypatch):
    import tae_trainer

    _guard_device(monkeypatch, tae_trainer)
    res = CliRunner().invoke(tae_trainer.train_video, ["--eval_clips", "-1"])
    assert res.exit_code == 2, (res.exit_code, res.output, res.exception)
    assert "eval_clips" in res.output


def test_eval_clips_reaches_the_training_loop(monkeypatch):
    import tae_trainer

    seen = {}
    monkeypatch.setattr(tae_trainer, "_train_video", lambda *a, **k: seen.update(args=a, kw=k))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.delenv("RANK", raising=False)
    res = CliRunner().invoke(tae_trainer.train_video, ["--eval_clips", "3"])
    assert res.exit_code == 0, res.output
    assert seen["kw"] == {"eval_clips": 3}
    res = CliRunner().invoke(tae_trainer.train_video, [])
    assert res.exit_code == 0, res.output
    assert seen["kw"] == {}  # the default trains exactly as before


def test_held_out_clips_do_not_depend_on_seed_or_rank(monkeypatch):
    import vae_trainer
    from tae_trainer import EVAL_SEED

    sets = []
    for rank in ("0", "3"):
        monkeypatch.setenv("RANK", rank)
        sets.append(vae_trainer.SyntheticLoader(1, 16, seed=EVAL_SEED, n_distinct=2, frames=4).batches)
    assert all(torch.equal(a, b) for a, b in zip(*sets))
    assert sets[0][0].shape == (1, 3, 4, 16, 16) and not torch.equal(sets[0][0], sets[0][1])
