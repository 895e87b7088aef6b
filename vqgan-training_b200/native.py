"""ctypes binding of libvqb200.so (C ABI declared in include/vqb200.h).

This is the only place Python touches the native layer. Tensors are passed as raw device pointers
(`tensor.data_ptr()`) plus the current CUDA stream; shapes travel in plain C structs. There is no
fallback: if the shared library is missing or the device is not sm_90 (H100) every op raises.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libvqb200.so")

VQB_MAX_VIEWS = 16
VQB_MAX_TAPS = 16
VQB_MAX_VIEWS_3D = 8
VQB_MAX_TAPS_3D = 27
VQB_MAX_TAPS_3D_DGRAD = 64
EPI_BIAS, EPI_RES, EPI_RELU, EPI_MASK, EPI_STATS = 1, 2, 4, 8, 16


class VqbView(C.Structure):
    _fields_ = [("offset", C.c_int64), ("Wv", C.c_int32), ("Hv", C.c_int32), ("Nv", C.c_int32), ("_pad", C.c_int32),
                ("sw", C.c_int64), ("sh", C.c_int64), ("sn", C.c_int64)]


class VqbTap(C.Structure):
    _fields_ = [("view", C.c_int32), ("dw", C.c_int32), ("dh", C.c_int32), ("_pad", C.c_int32)]


class VqbConvDesc(C.Structure):
    _fields_ = [("C", C.c_int32), ("Cout", C.c_int32), ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("nviews", C.c_int32), ("ntaps", C.c_int32), ("flags", C.c_int32), ("out_f32", C.c_int32),
                ("_pad", C.c_int32), ("on", C.c_int64), ("oh", C.c_int64), ("ow", C.c_int64), ("oc", C.c_int64),
                ("views", VqbView * VQB_MAX_VIEWS), ("taps", VqbTap * VQB_MAX_TAPS)]


class VqbWgradDesc(C.Structure):
    _fields_ = [("C", C.c_int32), ("Cout", C.c_int32), ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("nviews", C.c_int32), ("ntaps", C.c_int32), ("ksplit", C.c_int32), ("ld_override", C.c_int64),
                ("col_offset", C.c_int64), ("dy_view", VqbView),
                ("views", VqbView * VQB_MAX_VIEWS), ("taps", VqbTap * VQB_MAX_TAPS)]


class VqbPackJob(C.Structure):
    _fields_ = [("w", C.c_void_p), ("out", C.c_void_p), ("tapmap", C.c_void_p), ("Cout", C.c_int32), ("Cin", C.c_int32),
                ("T", C.c_int32), ("nslots", C.c_int32), ("transpose", C.c_int32), ("Kpad", C.c_int32),
                ("fold", C.c_int32), ("sg", C.c_int32), ("ld_g", C.c_int32), ("ld_r", C.c_int32),
                ("first_block", C.c_int32), ("w_bf16", C.c_int32)]


class VqbView3d(C.Structure):
    _fields_ = [("offset", C.c_int64), ("Wv", C.c_int32), ("Hv", C.c_int32), ("Tv", C.c_int32), ("Nv", C.c_int32),
                ("sw", C.c_int64), ("sh", C.c_int64), ("st", C.c_int64), ("sn", C.c_int64)]


class VqbTap3d(C.Structure):
    _fields_ = [("view", C.c_int32), ("dw", C.c_int32), ("dh", C.c_int32), ("dt", C.c_int32)]


class VqbConv3dDesc(C.Structure):
    _fields_ = [("C", C.c_int32), ("Cout", C.c_int32), ("N", C.c_int32), ("T", C.c_int32), ("H", C.c_int32),
                ("W", C.c_int32), ("nviews", C.c_int32), ("ntaps", C.c_int32), ("flags", C.c_int32),
                ("out_f32", C.c_int32), ("on", C.c_int64), ("ot", C.c_int64), ("oh", C.c_int64), ("ow", C.c_int64),
                ("oc", C.c_int64), ("views", VqbView3d * VQB_MAX_VIEWS_3D), ("taps", VqbTap3d * VQB_MAX_TAPS_3D)]


class VqbConv3dDgradDesc(C.Structure):
    _fields_ = [("C", C.c_int32), ("Cout", C.c_int32), ("N", C.c_int32), ("T", C.c_int32), ("H", C.c_int32),
                ("W", C.c_int32), ("nviews", C.c_int32), ("ntaps", C.c_int32), ("flags", C.c_int32),
                ("out_f32", C.c_int32), ("on", C.c_int64), ("ot", C.c_int64), ("oh", C.c_int64), ("ow", C.c_int64),
                ("oc", C.c_int64), ("views", VqbView3d * VQB_MAX_VIEWS_3D),
                ("taps", VqbTap3d * VQB_MAX_TAPS_3D_DGRAD)]


class VqbWgrad3dDesc(C.Structure):
    _fields_ = [("C", C.c_int32), ("Cout", C.c_int32), ("N", C.c_int32), ("T", C.c_int32), ("H", C.c_int32),
                ("W", C.c_int32), ("nviews", C.c_int32), ("ntaps", C.c_int32), ("ksplit", C.c_int32),
                ("_pad", C.c_int32), ("ld_override", C.c_int64), ("col_offset", C.c_int64), ("dy_view", VqbView3d),
                ("views", VqbView3d * VQB_MAX_VIEWS_3D), ("taps", VqbTap3d * VQB_MAX_TAPS_3D)]


class VqbAdamwGroup(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("weight_decay", C.c_float), ("step", C.c_int32)]


_lib = None


def lib_path() -> str:
    return _LIB_PATH


def load():
    """Loads libvqb200.so (building is the job of build_native.py / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            f"{_LIB_PATH} is missing: run `python vqgan-training_b200/build_native.py` (nvcc, sm_90a). "
            "There is no CPU / PyTorch fallback for the hot path.")
    L = C.CDLL(_LIB_PATH)
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
    sigs = {
        "vqb_last_error": (C.c_char_p, []),
        "vqb_version": (i32, []),
        "vqb_device_ok": (i32, []),
        "vqb_kernel_launch_count": (i32, []),
        "vqb_wgrad_cols": (i32, [i32, i32]),
        "vqb_conv_gemm": (i32, [C.POINTER(VqbConvDesc), vp, vp, vp, vp, vp, vp, vp, vp]),
        "vqb_wgrad_gemm": (i32, [C.POINTER(VqbWgradDesc), vp, vp, vp, vp]),
        "vqb_pack_weights": (i32, [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp]),
        "vqb_nchw_to_nhwc": (i32, [vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]),
        "vqb_nhwc_to_nchw": (i32, [vp, vp, i32, i32, i32, i32, i32, vp, vp]),
        "vqb_gn_silu_fwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, f32, i32, vp]),
        "vqb_gn_silu_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp]),
        "vqb_wavelet_fwd": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
        "vqb_colsum": (i32, [vp, vp, i64, i32, vp]),
        "vqb_wgrad_reduce": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp]),
        "vqb_maxpool2_fwd": (i32, [vp, vp, i32, i32, i32, i32, vp]),
        "vqb_maxpool2_bwd": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
        "vqb_lpips_tail_fwd": (i32, [vp, vp, vp, vp, i32, i32, i32, vp]),
        "vqb_lpips_tail_bwd": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, vp]),
        "vqb_lpips_tail_fwd_dropout": (i32, [vp, vp, vp, vp, i32, i32, i32, C.c_uint64, vp]),
        "vqb_lpips_tail_bwd_dropout": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, C.c_uint64, vp]),
        "vqb_lpips_dropout_mask": (i32, [C.c_uint64, i32, i32, i32, vp, vp]),
        "vqb_attn_fwd": (i32, [vp, vp, vp, i32, i32, i32, vp]),
        "vqb_attn_bwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, vp]),
        "vqb_vq_argmin": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, vp]),
        "vqb_nchw_to_nhwc_pad": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp]),
        "vqb_nhwc_to_nchw_pad": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp]),
        "vqb_gn_silu_fwd_pre": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, f32, i32, vp]),
        "vqb_conv_stats_ok": (i32, [C.POINTER(VqbConvDesc)]),
        "vqb_pack_weights_fold": (i32, [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp]),
        "vqb_wgrad_reduce_fold": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp]),
        "vqb_adamw_flat": (i32, [vp, vp, vp, vp, vp, i64, i32, C.POINTER(VqbAdamwGroup), f32, vp]),
        "vqb_pack_weights_multi": (i32, [vp, i32, i32, vp]),
        "vqb_adamw_fill_record": (i32, [i32, C.POINTER(VqbAdamwGroup), vp]),
        "vqb_adamw_flat_dev": (i32, [vp, vp, vp, vp, vp, i64, vp, f32, vp]),
        "vqb_adamw_ema_flat_dev": (i32, [vp, vp, vp, vp, vp, vp, i64, vp, vp, f32, vp]),
        "vqb_pack_weights_bf16": (i32, [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp]),
        "vqb_pack_weights_fold_bf16": (i32, [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp]),
        "vqb_nchw_to_nhwc_bf16": (i32, [vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]),
        "vqb_nchw_to_nhwc_pad_bf16": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp]),
        "vqb_nhwc_to_nchw_bf16": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
        "vqb_wavelet_fwd_bf16": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
        "vqb_conv3d_gemm": (i32, [C.POINTER(VqbConv3dDesc), vp, vp, vp, vp, vp, vp]),
        "vqb_attn_fwd_hd": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
        "vqb_gauss_reparam": (i32, [vp, vp, vp, i32, i32, i64, i32, vp]),
        "vqb_conv3d_dgrad_gemm": (i32, [C.POINTER(VqbConv3dDgradDesc), vp, vp, vp, vp]),
        "vqb_wgrad3d_gemm": (i32, [C.POINTER(VqbWgrad3dDesc), vp, vp, vp, vp]),
        "vqb_attn_bwd_hd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
        "vqb_gauss_reparam_bwd": (i32, [vp, vp, vp, vp, i32, i32, i64, vp]),
        "vqb_gn_silu_apply": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
        "vqb_ncthw_frames_to_nhwc_pad": (i32, [vp, vp] + [i32] * 7 + [vp, i32, vp, vp, vp]),
        "vqb_ncthw_frames_to_nhwc_pad_bf16": (i32, [vp, vp] + [i32] * 7 + [vp, i32, vp, vp, vp]),
        "vqb_ncthw_frames_to_nhwc": (i32, [vp, vp] + [i32] * 6 + [vp, i32, vp, vp, vp]),
        "vqb_ncthw_frames_to_nhwc_bf16": (i32, [vp, vp] + [i32] * 6 + [vp, i32, vp, vp, vp]),
        "vqb_nhwc_pad_frames_to_ncthw": (i32, [vp, vp] + [i32] * 7 + [vp, i32, vp, vp]),
        "vqb_nhwc_frames_to_ncthw": (i32, [vp, vp] + [i32] * 6 + [vp, i32, vp, vp]),
        "vqb_leaky_relu_fwd": (i32, [vp, vp, i64, vp]),
        "vqb_leaky_relu_bwd": (i32, [vp, vp, vp, i64, vp]),
        "vqb_psnr_ssim": (i32, [vp, vp] + [i32] * 6 + [f32, f32, vp, vp, vp, i64, vp]),
        "vqb_tile_blend": (i32, [vp, i32, vp, vp] + [i32] * 11 + [vp, vp, vp] + [i32] * 6 + [vp]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(L, name, None)
        if fn is None:
            continue  # optional symbols are checked by tests/test_abi.py against the header
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().vqb_last_error().decode(errors="replace")
        raise RuntimeError(f"libvqb200 {what} failed (code {rc}): {msg}")


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t) -> int:
    return 0 if t is None else t.data_ptr()


def launch_count() -> int:
    return load().vqb_kernel_launch_count()


def dense_view3d(N: int, T: int, H: int, W: int, Cs: int) -> VqbView3d:
    """Dense NTHWC view with channel row stride Cs."""
    return VqbView3d(offset=0, Wv=W, Hv=H, Tv=T, Nv=N, sw=Cs, sh=W * Cs, st=H * W * Cs, sn=T * H * W * Cs)


def dense_view(N: int, H: int, W: int, Cs: int) -> VqbView:
    """Dense NHWC view with channel row stride Cs."""
    return VqbView(offset=0, Wv=W, Hv=H, Nv=N, _pad=0, sw=Cs, sh=W * Cs, sn=H * W * Cs)
