"""CPU: libvqb200.so loads without a GPU and exports every symbol declared in include/vqb200.h; argument validation
of the compute entry points fails loudly (no CPU fallback) when no sm_90 device is present."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vqb200.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vqb_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    import native

    if not os.path.exists(native.lib_path()):
        import build_native

        build_native.build()
    return native.load()


def test_header_declares_entry_points():
    syms = declared_symbols()
    assert "vqb_conv_gemm" in syms and "vqb_wgrad_gemm" in syms and len(syms) >= 20


def test_library_exports_every_declared_symbol(lib):
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"include/vqb200.h declares symbols the library does not export: {missing}"


def test_version_and_error_channel(lib):
    assert lib.vqb_version() >= 100
    lib.vqb_last_error.restype = ctypes.c_char_p
    assert isinstance(lib.vqb_last_error(), bytes)


def test_compute_fails_loudly_without_device(lib):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    import native

    assert lib.vqb_device_ok() == 0
    d = native.VqbConvDesc()
    d.C, d.Cout, d.N, d.H, d.W, d.nviews, d.ntaps = 64, 64, 1, 8, 8, 1, 1
    d.on, d.oh, d.ow, d.oc = 8 * 8 * 64, 8 * 64, 64, 1
    buf = (ctypes.c_uint8 * 65536)()
    p = ctypes.addressof(buf)
    rc = lib.vqb_conv_gemm(d, p, p, None, None, None, p, None, None)
    assert rc == -2  # VQB_ENODEVICE: there is no CPU path
    assert b"sm_90" in lib.vqb_last_error()
    assert lib.vqb_conv_gemm(None, None, None, None, None, None, None, None, None) == -1  # VQB_EINVAL


def test_struct_layout_matches_header(lib):
    """ctypes mirrors of the C structs must have the sizes the compiler gives them (checked via sizeof constants)."""
    import native

    assert ctypes.sizeof(native.VqbView) == 48
    assert ctypes.sizeof(native.VqbTap) == 16
    assert ctypes.sizeof(native.VqbConvDesc) == 40 + 32 + 16 * 48 + 16 * 16
    assert ctypes.sizeof(native.VqbWgradDesc) == 32 + 16 + 48 + 16 * 48 + 16 * 16
