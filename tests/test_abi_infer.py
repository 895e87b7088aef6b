"""CPU: the bf16 inference entry points of include/vqb200.h validate their arguments (VQB_EINVAL) and, given valid
arguments, fail with VQB_ENODEVICE when no sm_90 device is present (there is no CPU path)."""
import ctypes
import os

import pytest
import torch

EINVAL, ENODEVICE = -1, -2


@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    return native.load()


def calls(p):
    """(name, call with valid arguments, call with invalid arguments) for every bf16 inference entry point."""
    return [
        ("vqb_pack_weights_bf16",
         lambda L: L.vqb_pack_weights_bf16(p, p, 64, 32, 9, 9, p, 0, 32, None),
         lambda L: L.vqb_pack_weights_bf16(p, p, 64, 32, 9, 9, p, 0, 20, None)),  # Kpad not a multiple of 8
        ("vqb_pack_weights_fold_bf16",
         lambda L: L.vqb_pack_weights_fold_bf16(p, p, 64, 32, 9, 4, p, 1, 64, None),
         lambda L: L.vqb_pack_weights_fold_bf16(None, p, 64, 32, 9, 4, p, 1, 64, None)),
        ("vqb_nchw_to_nhwc_bf16",
         lambda L: L.vqb_nchw_to_nhwc_bf16(p, p, 1, 3, 8, 8, 8, None, None, None),
         lambda L: L.vqb_nchw_to_nhwc_bf16(p, p, 1, 9, 8, 8, 8, None, None, None)),  # Cpad < C
        ("vqb_nchw_to_nhwc_pad_bf16",
         lambda L: L.vqb_nchw_to_nhwc_pad_bf16(p, p, 1, 3, 8, 8, 8, 1, None, None, None),
         lambda L: L.vqb_nchw_to_nhwc_pad_bf16(p, p, 1, 3, 8, 8, 8, -1, None, None, None)),
        ("vqb_nhwc_to_nchw_bf16",
         lambda L: L.vqb_nhwc_to_nchw_bf16(p, p, 1, 3, 8, 8, 8, None),
         lambda L: L.vqb_nhwc_to_nchw_bf16(p, None, 1, 3, 8, 8, 8, None)),
        ("vqb_wavelet_fwd_bf16",
         lambda L: L.vqb_wavelet_fwd_bf16(p, p, p, 1, 3, 8, 8, 16, None),
         lambda L: L.vqb_wavelet_fwd_bf16(p, p, p, 1, 3, 7, 8, 16, None)),  # odd H
    ]


def test_bf16_entry_points_are_declared_and_exported(lib):
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vqb200.h")).read()
    for name, _, _ in calls(0):
        assert f"int {name}(" in hdr, name
        assert hasattr(lib, name), name


def test_bf16_entry_points_fail_without_device(lib):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib.vqb_last_error.restype = ctypes.c_char_p
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.addressof(buf)
    for name, good, bad in calls(p):
        assert bad(lib) == EINVAL, name
        assert good(lib) == ENODEVICE, name
        assert b"sm_90" in lib.vqb_last_error(), name


def test_pack_job_carries_the_source_dtype():
    """VqbPackJob keeps its size (the multi-pack kernel reads a device array of them); the former pad word is w_bf16."""
    import native

    assert ctypes.sizeof(native.VqbPackJob) == 3 * 8 + 12 * 4
    assert [f for f, _ in native.VqbPackJob._fields_][-1] == "w_bf16"


def test_unsupported_parameter_dtype_is_refused_on_the_host():
    import ops

    for dt in (torch.float16, torch.float64):
        with pytest.raises(RuntimeError, match=str(dt)):
            ops.check_master_dtype(torch.zeros(2, dtype=dt))
    ops.check_master_dtype(torch.zeros(2, dtype=torch.bfloat16))
    ops.check_master_dtype(torch.zeros(2))
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.inference_only(torch.zeros(2, dtype=torch.bfloat16))
