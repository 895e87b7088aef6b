"""CPU: the C ABI of the LPIPS tail, dropout-mask, VQ search and fused AdamW entry points. Without a CUDA device, bad
arguments fail with VQB_EINVAL and a message that names the entry point, and valid ones with VQB_ENODEVICE: every
argument is checked before the device, and no width the kernels cannot serve reaches a launch (the LPIPS backward once
took C = 320, 384 and 448 and left channels 256..C-1 of df0 unwritten; C = 0 divided by zero on the host).
vqb_adamw_fill_record is a host function: its 28-float record layout is checked here."""
import ctypes
import math
import os
import struct

import pytest
import torch

EINVAL, ENODEVICE = -1, -2
BAD_LPIPS_C = (0, 8, 192, 320, 384, 448, 576)
GOOD_LPIPS_C = (64, 128, 256, 512)


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


def _buf():
    """A 16-byte aligned host address (never dereferenced: every call below fails before it touches memory)."""
    buf = (ctypes.c_uint8 * 4096)()
    return buf, (ctypes.addressof(buf) + 15) // 16 * 16


def _expect(L, name, rc, code):
    err = L.vqb_last_error()
    assert rc == code, (name, rc, err)
    assert name.encode() in err, (name, err)
    if code == ENODEVICE:
        assert b"sm_90" in err, err


def _lpips_calls(L, p):
    """name -> call(f0, f1, w, out_or_g, df0, N, HW, C) for the four LPIPS tail entry points."""
    seed = 2 ** 64 - 1
    return {
        "vqb_lpips_tail_fwd": lambda a, b, w, o, d, N, HW, C: L.vqb_lpips_tail_fwd(a, b, w, o, N, HW, C, None),
        "vqb_lpips_tail_fwd_dropout":
            lambda a, b, w, o, d, N, HW, C: L.vqb_lpips_tail_fwd_dropout(a, b, w, o, N, HW, C, seed, None),
        "vqb_lpips_tail_bwd": lambda a, b, w, g, d, N, HW, C: L.vqb_lpips_tail_bwd(a, b, w, g, d, N, HW, C, None),
        "vqb_lpips_tail_bwd_dropout":
            lambda a, b, w, g, d, N, HW, C: L.vqb_lpips_tail_bwd_dropout(a, b, w, g, d, N, HW, C, seed, None),
    }


def test_lpips_tail_entry_points_validate_then_need_a_device(lib, no_device):
    _keep, p = _buf()
    for name, call in _lpips_calls(lib, p).items():
        for C in BAD_LPIPS_C:
            _expect(lib, name, call(p, p, p, p, p, 3, 97, C), EINVAL)
            assert f"C={C}".encode() in lib.vqb_last_error(), (name, C)
        for N, HW in ((0, 97), (-1, 97), (3, 0), (3, -5)):
            _expect(lib, name, call(p, p, p, p, p, N, HW, 64), EINVAL)
        for k in range(5):  # each pointer null in turn (the forward ignores the fifth)
            if k == 4 and "fwd" in name:
                continue
            args = [p] * 5
            args[k] = None
            _expect(lib, name, call(*args, 3, 97, 64), EINVAL)
        for C in GOOD_LPIPS_C:
            _expect(lib, name, call(p, p, p, p, p, 3, 97, C), ENODEVICE)
        _expect(lib, name, call(p, p, p, p, p, 1, 1, 512), ENODEVICE)


def test_lpips_dropout_mask_validates_then_needs_a_device(lib, no_device):
    _keep, p = _buf()
    name = "vqb_lpips_dropout_mask"
    for seed, N, HW, C, m in ((0, 3, 5, 8, None), (1, 3, 5, 12, p), (1, 3, 5, 0, p), (1, 0, 5, 8, p),
                              (1, 3, -1, 8, p)):
        _expect(lib, name, lib.vqb_lpips_dropout_mask(seed, N, HW, C, m, None), EINVAL)
    for seed in (0, 1, 2 ** 64 - 1):
        _expect(lib, name, lib.vqb_lpips_dropout_mask(seed, 3, 5, 8, p, None), ENODEVICE)


def test_vq_argmin_validates_then_needs_a_device(lib, no_device):
    _keep, p = _buf()
    name = "vqb_vq_argmin"
    f = lib.vqb_vq_argmin
    for M, K, D in ((100, 33, 0), (100, 33, 257), (100, 33, -1), (0, 33, 16), (100, 0, 16)):
        _expect(lib, name, f(p, p, p, p, p, M, K, D, None), EINVAL)
    for k in range(4):  # z, e, idx, zq must be given; sqerr is optional
        args = [p] * 5
        args[k] = None
        _expect(lib, name, f(*args, 100, 33, 16, None), EINVAL)
    for M, K, D in ((1, 1, 1), (20000, 1025, 16), (100, 300, 256), (5, 33, 255)):
        _expect(lib, name, f(p, p, p, p, p, M, K, D, None), ENODEVICE)
        _expect(lib, name, f(p, p, p, p, None, M, K, D, None), ENODEVICE)


def _groups(n, step=1):
    import native

    arr = (native.VqbAdamwGroup * 4)()
    for i in range(n):
        arr[i].lr, arr[i].beta1, arr[i].beta2 = 1e-3 * (i + 1), 0.9 - 0.05 * i, 0.95 + 0.01 * i
        arr[i].eps, arr[i].weight_decay, arr[i].step = 1e-8 * 10 ** i, 1e-3 * i, step + 3 * i
    return arr


def test_adamw_entry_points_validate_then_need_a_device(lib, no_device):
    _keep, p = _buf()
    gr = _groups(4)
    flat, dev = lib.vqb_adamw_flat, lib.vqb_adamw_flat_dev
    for k in range(5):  # params, grads, exp_avg, exp_avg_sq, chunk_group
        args = [p] * 5
        args[k] = None
        _expect(lib, "vqb_adamw_flat", flat(*args, 3, 4, gr, 1.0, None), EINVAL)
        _expect(lib, "vqb_adamw_flat_dev", dev(*args, 3, p, 1.0, None), EINVAL)
    _expect(lib, "vqb_adamw_flat", flat(p, p, p, p, p, 3, 4, None, 1.0, None), EINVAL)
    _expect(lib, "vqb_adamw_flat_dev", dev(p, p, p, p, p, 3, None, 1.0, None), EINVAL)
    for k, off in ((0, 4), (1, 8), (2, 12), (3, 4)):  # one fp32 buffer off its 16-byte alignment
        args = [p] * 4
        args[k] = p + off
        _expect(lib, "vqb_adamw_flat", flat(*args, p, 3, 4, gr, 1.0, None), EINVAL)
        _expect(lib, "vqb_adamw_flat_dev", dev(*args, p, 3, p, 1.0, None), EINVAL)
    for ng in (0, 5, -1):
        _expect(lib, "vqb_adamw_flat", flat(p, p, p, p, p, 3, ng, gr, 1.0, None), EINVAL)
    _expect(lib, "vqb_adamw_flat", flat(p, p, p, p, p, 3, 4, _groups(4, step=0), 1.0, None), EINVAL)
    for ng in (1, 4):
        _expect(lib, "vqb_adamw_flat", flat(p, p, p, p, p, 3001, ng, gr, 0.37, None), ENODEVICE)
    _expect(lib, "vqb_adamw_flat_dev", dev(p, p, p, p, p, 3001, p, 0.37, None), ENODEVICE)


@pytest.mark.parametrize("ngroups", [1, 2, 3, 4])
def test_adamw_fill_record_layout(lib, ngroups):
    """28 floats: lr, beta1, beta2, eps, wd, bc1, bc2_sqrt, each x4; groups past ngroups repeat group 0; the bias
    corrections are 1 - beta1^step and sqrt(1 - beta2^step) in double, rounded once to fp32."""
    gr = _groups(ngroups, step=7)
    rec = (ctypes.c_float * 28)()
    assert lib.vqb_adamw_fill_record(ngroups, gr, rec) == 0, lib.vqb_last_error()
    f32 = lambda x: struct.unpack("f", struct.pack("f", x))[0]  # noqa: E731
    for i in range(4):
        s = gr[i if i < ngroups else 0]
        want = [s.lr, s.beta1, s.beta2, s.eps, s.weight_decay, f32(1.0 - float(s.beta1) ** s.step),
                f32(math.sqrt(1.0 - float(s.beta2) ** s.step))]
        got = [rec[k * 4 + i] for k in range(7)]
        assert got == want, (ngroups, i, got, want)


def test_adamw_fill_record_rejects_bad_arguments(lib):
    rec = (ctypes.c_float * 28)()
    gr = _groups(4)
    for args in ((0, gr, rec), (5, gr, rec), (2, None, rec), (2, gr, None), (2, _groups(2, step=0), rec)):
        _expect(lib, "vqb_adamw_fill_record", lib.vqb_adamw_fill_record(*args), EINVAL)
