"""CPU: the 3-D PatchGAN discriminator of video training (tae_disc.PatchDiscriminator3D). The oracle's output shapes;
parameter names and state_dict round trips between the oracle and the native module; host refusals before any launch;
the C ABI of the LeakyReLU activation code of the GroupNorm entry points and of vqb_leaky_relu_fwd / _bwd (VQB_EINVAL
for bad arguments, VQB_ENODEVICE for valid ones without an sm_90 device); the train_video options of the clip
discriminator and their refusal before any device work."""
import ctypes
import os

import pytest
import torch
import torch.distributed as dist
from click.testing import CliRunner

from oracle import clip_disc_oracle as CDO

EINVAL, ENODEVICE = -1, -2


@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    return native.load()


@pytest.mark.parametrize("T,H,W,n_layers", [(2, 2, 2, 1), (8, 48, 80, 3), (16, 32, 32, 4), (4, 8, 12, 2),
                                            (8, 16, 16, 1)])
def test_oracle_output_shapes(T, H, W, n_layers):
    d = CDO.PatchDiscriminator3D(ch=32, n_layers=n_layers)
    x = torch.randn(2, 3, T, H, W)
    f = 2 ** n_layers
    with torch.no_grad():
        y = d(x)
        yf = CDO.forward(d.state_dict(), x, n_layers)
    assert y.shape == (2, (T // f) * (H // f) * (W // f))
    torch.testing.assert_close(yf, y, rtol=1e-5, atol=1e-6)


def test_oracle_channel_plan_and_init():
    assert CDO.channel_plan(64, 3) == [(3, 64, 2), (64, 128, 2), (128, 256, 2), (256, 512, 1), (512, 1, 1)]
    assert CDO.channel_plan(32, 5)[-2:] == [(256, 256, 1), (256, 1, 1)]  # m_i = min(2^i, 8)
    torch.manual_seed(0)
    d = CDO.PatchDiscriminator3D(ch=64, n_layers=3)
    w = d.mid.conv.weight.detach()
    assert abs(float(w.std()) - 0.02) < 1e-3 and abs(float(w.mean())) < 1e-3
    assert not d.conv_in.bias.any() and not d.conv_out.bias.any() and d.mid.conv.bias is None
    assert bool((d.down[0].norm.weight == 1).all()) and not d.down[0].norm.bias.any()


@pytest.mark.parametrize("ch,n_layers", [(32, 1), (64, 2), (64, 3), (32, 5)])
def test_state_dicts_load_both_ways(ch, n_layers):
    import tae_disc

    o = CDO.PatchDiscriminator3D(ch=ch, n_layers=n_layers)
    m = tae_disc.PatchDiscriminator3D(ch=ch, n_layers=n_layers)
    assert list(o.state_dict()) == list(m.state_dict())
    assert [n for n, _ in o.named_parameters()] == [n for n, _ in m.named_parameters()]
    m.load_state_dict(o.state_dict(), strict=True)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in o.state_dict().items())
    torch.manual_seed(3)
    m2 = tae_disc.PatchDiscriminator3D(ch=ch, n_layers=n_layers)
    o.load_state_dict(m2.state_dict(), strict=True)
    assert all(torch.equal(o.state_dict()[k], v) for k, v in m2.state_dict().items())


def test_native_init_matches_the_oracle_distribution():
    import tae_disc

    torch.manual_seed(0)
    m = tae_disc.PatchDiscriminator3D(ch=64, n_layers=3)
    assert abs(float(m.mid.conv.weight.std()) - 0.02) < 1e-3
    assert not m.conv_in.bias.any() and not m.conv_out.bias.any()
    assert bool((m.mid.norm.weight == 1).all()) and not m.mid.norm.bias.any()


@pytest.mark.parametrize("make, shape, match", [
    (dict(ch=32, n_layers=3), (1, 3, 8, 16, 12), r"divisible by 8.*\(1, 3, 8, 16, 12\)"),
    (dict(ch=32, n_layers=2), (1, 3, 6, 16, 16), r"divisible by 4.*\(1, 3, 6, 16, 16\)"),
    (dict(ch=32, n_layers=1), (1, 3, 3, 16, 16), "divisible by 2"),
    (dict(ch=32, n_layers=1), (3, 16, 16, 16), r"\[B, 3, T, H, W\]"),
    (dict(ch=32, n_layers=1), (1, 4, 2, 16, 16), r"\[B, 3, T, H, W\]"),
    (dict(ch=48, n_layers=1), None, "multiple of 32"),
    (dict(ch=512, n_layers=1), None, "multiple of 32 up to 256"),
    (dict(ch=32, n_layers=0), None, "n_layers"),
])
def test_host_refusals_launch_nothing(lib, make, shape, match):
    import native
    import tae_disc

    n0 = native.launch_count()
    with pytest.raises(ValueError, match=match):
        d = tae_disc.PatchDiscriminator3D(**make)
        with torch.no_grad():
            d(torch.zeros(shape))
    assert native.launch_count() == n0


def test_training_needs_the_opt_in():
    import tae_disc

    d = tae_disc.PatchDiscriminator3D(ch=32, n_layers=1)
    with pytest.raises(RuntimeError, match="enable_training"):
        d(torch.zeros(1, 3, 2, 8, 8))


# ------------------------------------------------------------------------------------------------ C ABI
def test_leaky_entry_points_are_declared_and_exported(lib):
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vqb200.h")).read()
    assert "int vqb_leaky_relu_fwd(const void* x, void* y, int64_t n, void* stream);" in hdr
    assert "int vqb_leaky_relu_bwd(const void* y, const void* dy, void* dx, int64_t n, void* stream);" in hdr
    assert hasattr(lib, "vqb_leaky_relu_fwd") and hasattr(lib, "vqb_leaky_relu_bwd")


def _gn_calls(p, act):
    return {
        "vqb_gn_silu_fwd": lambda L: L.vqb_gn_silu_fwd(p, p, p, p, p, p, 2, 37, 64, 32, 1e-6, act, None),
        "vqb_gn_silu_fwd_pre": lambda L: L.vqb_gn_silu_fwd_pre(p, p, p, p, p, p, 2, 37, 64, 32, 1e-6, act, None),
        "vqb_gn_silu_bwd": lambda L: L.vqb_gn_silu_bwd(p, p, None, p, p, p, p, p, p, p, 2, 37, 64, 32, act, None,
                                                       None),
    }


def test_activation_codes_of_the_groupnorm_entry_points(lib):
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    for act in (3, -1, 7):
        for name, call in _gn_calls(p, act).items():
            assert call(lib) == EINVAL, (name, act)
            err = lib.vqb_last_error()
            assert name.encode() in err and f"activation code {act}".encode() in err, (name, err)
    # the recompute entry point keeps taking swish / none only
    for act in (2, 3):
        assert lib.vqb_gn_silu_apply(p, p, p, p, p, 1, 64, 64, 32, act, None) == EINVAL
    if torch.cuda.is_available():
        return
    for act in (0, 1, 2):
        for name, call in _gn_calls(p, act).items():
            assert call(lib) == ENODEVICE, (name, act)
            assert b"sm_90" in lib.vqb_last_error()


def test_leaky_relu_entry_points_validate_then_need_a_device(lib):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    fwd, bwd = lib.vqb_leaky_relu_fwd, lib.vqb_leaky_relu_bwd
    bads = [
        ("vqb_leaky_relu_fwd", lambda: fwd(None, p, 64, None)),
        ("vqb_leaky_relu_fwd", lambda: fwd(p, None, 64, None)),
        ("vqb_leaky_relu_fwd", lambda: fwd(p, p, 0, None)),
        ("vqb_leaky_relu_fwd", lambda: fwd(p, p, -8, None)),
        ("vqb_leaky_relu_fwd", lambda: fwd(p, p, 60, None)),      # n % 8
        ("vqb_leaky_relu_fwd", lambda: fwd(p + 2, p, 64, None)),  # x misaligned
        ("vqb_leaky_relu_fwd", lambda: fwd(p, p + 8, 64, None)),  # y misaligned
        ("vqb_leaky_relu_bwd", lambda: bwd(None, p, p, 64, None)),
        ("vqb_leaky_relu_bwd", lambda: bwd(p, None, p, 64, None)),
        ("vqb_leaky_relu_bwd", lambda: bwd(p, p, None, 64, None)),
        ("vqb_leaky_relu_bwd", lambda: bwd(p, p, p, 12, None)),
        ("vqb_leaky_relu_bwd", lambda: bwd(p, p + 4, p, 64, None)),
        ("vqb_leaky_relu_bwd", lambda: bwd(p, p, p + 2, 64, None)),
    ]
    for i, (name, bad) in enumerate(bads):
        assert bad() == EINVAL, i
        assert name.encode() in lib.vqb_last_error(), i
    for n in (8, 64, 1 << 33):
        assert fwd(p, p, n, None) == ENODEVICE
        assert b"vqb_leaky_relu_fwd" in lib.vqb_last_error() and b"sm_90" in lib.vqb_last_error()
        assert bwd(p, p, p, n, None) == ENODEVICE


# ------------------------------------------------------------------------------------------------ trainer and CLI
def test_trainer_requires_a_clip_disc_learning_rate():
    import tae_trainer

    with pytest.raises(ValueError, match="lr_clip_disc"):
        tae_trainer.VideoTrainer(torch.nn.Linear(1, 1), None, None, lr_vae=1e-4, clip_discriminator=object())


def test_help_lists_the_clip_disc_options():
    import tae_trainer

    res = CliRunner().invoke(tae_trainer.train_video, ["--help"])
    assert res.exit_code == 0, res.output
    for o in ("--do_clip_ganloss", "--clip_disc_ch", "--clip_disc_layers", "--learning_rate_clip_disc"):
        assert o in res.output, o


def _parse(argv, monkeypatch):
    import tae_trainer

    seen = {}
    monkeypatch.setattr(tae_trainer, "_train_video", lambda *a, **k: seen.update(args=a, kw=k))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.delenv("RANK", raising=False)
    res = CliRunner().invoke(tae_trainer.train_video, argv)
    assert res.exit_code == 0, res.output
    return seen


def test_cli_parses_the_clip_disc_options(monkeypatch):
    base = ["--clip_frames", "8", "--resolution", "32", "--learning_rate_disc", "5e-4"]
    seen = _parse(base + ["--do_clip_ganloss", "--clip_disc_ch", "32", "--clip_disc_layers", "2",
                          "--learning_rate_clip_disc", "3e-4"], monkeypatch)
    assert seen["kw"] == {"clip_disc": (32, 2, 3e-4)}
    seen = _parse(base + ["--do_clip_ganloss"], monkeypatch)
    assert seen["kw"] == {"clip_disc": (64, 3, 5e-4)}  # defaults; the learning rate is --learning_rate_disc's
    seen = _parse(base + ["--clip_disc_ch", "48"], monkeypatch)  # ignored without --do_clip_ganloss
    assert seen["kw"] == {} and len(seen["args"]) == 22


@pytest.mark.parametrize("argv, match", [
    (["--do_clip_ganloss", "--clip_disc_ch", "48"], "clip_disc_ch"),
    (["--do_clip_ganloss", "--clip_disc_ch", "0"], "clip_disc_ch"),
    (["--do_clip_ganloss", "--clip_disc_ch", "512"], "clip_disc_ch"),
    (["--do_clip_ganloss", "--clip_disc_layers", "0"], "clip_disc_layers"),
    (["--do_clip_ganloss", "--clip_disc_layers", "5", "--clip_frames", "16"], "multiples of 32"),
    (["--do_clip_ganloss", "--clip_disc_layers", "3", "--clip_frames", "4", "--vae_ch_mult", "1,2"], "multiples of 8"),
    (["--do_clip_ganloss", "--clip_disc_ch", "x"], "clip_disc_ch"),
])
def test_bad_clip_disc_arguments_are_refused_before_device_work(argv, match, monkeypatch):
    import tae_trainer

    def device_work(*a, **k):
        raise AssertionError("device work before the arguments were checked")

    monkeypatch.setattr(torch.cuda, "is_available", device_work)
    monkeypatch.setattr(torch.cuda, "set_device", device_work)
    monkeypatch.setattr(dist, "init_process_group", device_work)
    monkeypatch.setattr(tae_trainer, "_train_video", device_work)
    res = CliRunner().invoke(tae_trainer.train_video, argv)
    assert res.exit_code == 2, (res.exit_code, res.output, res.exception)
    assert match in res.output
