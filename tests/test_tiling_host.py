"""CPU: tiled encode / decode without a GPU. The float64 oracle's planner and weights (oracle/tiling_oracle.py) have the
properties DESIGN.md section 7 row 27 states; tiling.py's planner and fp32 weight tables equal the oracle's bit for bit;
tiling.encode / tiling.decode refuse every bad call before anything launches; the C entry point vqb_tile_blend returns
VQB_EINVAL for bad arguments and VQB_ENODEVICE without a device; its translation unit compiles without ptxas spills."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import tiling_oracle as TO

EINVAL, ENODEVICE = -1, -2


# ---------------------------------------------------------------------------------------------------- planner
def _sweep(limit=28):
    for L in range(1, limit + 1):
        for O in range(L):
            for X in range(1, limit + 1):
                yield X, L, O


def test_oracle_plan_properties():
    for X, L, O in _sweep():
        starts, length = TO.plan_axis(X, L, O)
        n = len(starts)
        if X <= L:
            assert (starts, length) == ([0], X)
            continue
        assert length == L and starts[0] == 0 and starts[-1] + L == X, (X, L, O, starts)
        gaps = np.diff(starts)
        assert np.all(gaps > 0), (X, L, O, starts)  # strictly increasing
        assert np.all(gaps <= L - O), (X, L, O, starts)  # every realised overlap L - gap >= O, and no hole
        assert (n - 2) * (L - O) + L < X, (X, L, O, n)  # n - 1 tiles with stride <= L - O cannot reach X


@pytest.mark.parametrize("f", [1, 2, 8])
def test_grid_plans_are_multiples_of_f(f):
    for X, L, O in _sweep(16):
        a = TO.axis(X, L * f, O * f, f, decode=True)
        assert all(s % f == 0 for s in a["gstarts"]) and a["glen"] % f == 0 and a["gextent"] == X * f
        assert a["R"] == O * f
        e = TO.axis(X, L * f, O * f, f, decode=False)
        assert e["gstarts"] == e["starts"] and e["glen"] == e["length"] and e["R"] == O


def test_tiling_planner_equals_the_oracle():
    import tiling

    for X, L, O in _sweep():
        assert tiling.plan_axis(X, L, O) == TO.plan_axis(X, L, O), (X, L, O)


# ---------------------------------------------------------------------------------------------------- weights
@pytest.mark.parametrize("f", [1, 2, 8])
@pytest.mark.parametrize("decode", [True, False])
def test_weights_sum_to_one(f, decode):
    for X, L, O in _sweep(14):
        a = TO.axis(X, L * f, O * f, f, decode)
        total = np.zeros(a["gextent"])
        for s, w in zip(a["gstarts"], a["weights"]):
            assert np.all(w > 0)
            total[s:s + a["glen"]] += w
        np.testing.assert_allclose(total, 1.0, rtol=0, atol=1e-12, err_msg=str((X, L, O, f, decode)))


@pytest.mark.parametrize("X, L, O", [(10, 4, 2), (36, 8, 4), (5, 3, 1), (12, 6, 3)])
def test_exact_overlaps_are_the_linear_cross_fade(X, L, O):
    starts, _ = TO.plan_axis(X, L, O)
    assert np.all(np.diff(starts) == L - O) and 2 * O <= L  # every overlap is exactly R, two tiles per cell at most
    w = TO.axis_weights(starts, L, O)
    x = np.arange(L)
    up, down = (x + 0.5) / O, (L - x - 0.5) / O
    for k in range(len(starts)):
        ramp = np.minimum(np.minimum(1.0, up if k > 0 else 1.0), down if k < len(starts) - 1 else 1.0)
        np.testing.assert_allclose(w[k], ramp, rtol=0, atol=1e-15)


def test_zero_overlap_is_a_partition():
    w = TO.axis_weights([0, 4, 8], 4, 0)
    np.testing.assert_array_equal(w, np.ones((3, 4)))
    # an even spread can overlap tiles even with O = 0: the shared cells are averaged
    starts, L = TO.plan_axis(10, 4, 0)
    assert starts == [0, 3, 6]
    w = TO.axis_weights(starts, L, 0)
    np.testing.assert_array_equal(w[0], [1, 1, 1, 0.5])


@pytest.mark.parametrize("f", [1, 2, 8])
@pytest.mark.parametrize("decode", [True, False])
def test_tiling_tables_equal_the_oracle_bit_for_bit(f, decode):
    import tiling

    for X, L, O in _sweep(14):
        a = TO.axis(X, L * f, O * f, f, decode)
        t = tiling._Axis(X, L * f, O * f, f, decode)
        assert (t.gstarts, t.glen, t.gextent) == (a["gstarts"], a["glen"], a["gextent"])
        np.testing.assert_array_equal(t.table.numpy().view(np.int32), a["weights"].astype(np.float32).view(np.int32),
                                      err_msg=str((X, L, O, f, decode)))


def test_oracle_blend_of_constant_tiles_is_constant():
    axes = [TO.axis(6, 4, 2, 2, True), TO.axis(9, 8, 2, 2, True), TO.axis(11, 6, 4, 2, True)]
    import itertools

    outs = {idx: np.full((1, 2) + tuple(a["glen"] for a in axes), 3.0)
            for idx in itertools.product(*(range(len(a["gstarts"])) for a in axes))}
    np.testing.assert_allclose(TO.blend(outs, axes), 3.0, rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------------------------------- refusals
@pytest.fixture(scope="module")
def modules():
    import ae
    import tae

    tv = tae.TVAE(resolution=16, in_channels=3, ch=32, out_ch=3, ch_mult=[1, 2], num_res_blocks=1, z_channels=4)
    av = ae.VAE(32, 3, 32, 3, [1, 2], 1, 4, False, False, False)
    return {"tenc": tv.encoder, "tdec": tv.decoder, "aenc": av.encoder, "adec": av.decoder}


def _x(*shape, **kw):
    return torch.zeros(*shape, **kw)


T3, O3 = (4, 8, 8), (2, 2, 2)
REFUSALS = [
    ("encode with a decoder", "encode", "tdec", lambda: _x(1, 3, 4, 8, 8), T3, O3, TypeError),
    ("decode with an encoder", "decode", "aenc", lambda: _x(1, 4, 4, 4), (8, 8), (2, 2), TypeError),
    ("tae rank 4", "encode", "tenc", lambda: _x(1, 3, 8, 8), T3, O3, ValueError),
    ("ae rank 5", "decode", "adec", lambda: _x(1, 4, 2, 4, 4), (8, 8), (2, 2), ValueError),
    ("tile length", "encode", "tenc", lambda: _x(1, 3, 4, 8, 8), (8, 8), (2, 2), ValueError),
    ("overlap length", "decode", "tdec", lambda: _x(1, 4, 2, 4, 4), T3, (2, 2), ValueError),
    ("tile not ints", "decode", "adec", lambda: _x(1, 4, 4, 4), (8.0, 8.0), (2, 2), ValueError),
    ("tile not a multiple of f", "encode", "tenc", lambda: _x(1, 3, 4, 8, 8), (4, 7, 8), O3, ValueError),
    ("overlap not a multiple of f", "decode", "adec", lambda: _x(1, 4, 4, 4), (8, 8), (2, 3), ValueError),
    ("negative overlap", "decode", "tdec", lambda: _x(1, 4, 2, 4, 4), T3, (2, -2, 2), ValueError),
    ("zero tile", "decode", "tdec", lambda: _x(1, 4, 2, 4, 4), (0, 8, 8), (0, 2, 2), ValueError),
    ("overlap == tile", "encode", "aenc", lambda: _x(1, 3, 8, 8), (8, 8), (2, 8), ValueError),
    ("overlap > tile", "decode", "tdec", lambda: _x(1, 4, 2, 4, 4), T3, (6, 2, 2), ValueError),
    ("extent not a multiple of f", "encode", "tenc", lambda: _x(1, 3, 4, 8, 9), T3, O3, ValueError),
    ("odd image extent", "encode", "aenc", lambda: _x(1, 3, 7, 8), (4, 4), (2, 2), ValueError),
    ("empty batch", "decode", "adec", lambda: _x(0, 4, 4, 4), (8, 8), (2, 2), ValueError),
    ("input requires grad", "decode", "tdec", lambda: _x(1, 4, 2, 4, 4, requires_grad=True), T3, O3, RuntimeError),
    ("grad mode", "encode", "aenc", lambda: _x(1, 3, 8, 8), (4, 4), (2, 2), RuntimeError),
]


@pytest.mark.parametrize("what, fn, mod, make, tile, overlap, exc", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_bad_calls_are_refused_before_any_launch(modules, what, fn, mod, make, tile, overlap, exc):
    import native
    import tiling

    native.load()
    n0 = native.launch_count()
    with pytest.raises(exc, match=r"f = \d|expected a|inference only"):
        getattr(tiling, fn)(modules[mod], make(), tile=tile, overlap=overlap)
    assert native.launch_count() == n0


def test_grad_mode_refusal_names_no_grad(modules):
    import tiling

    with pytest.raises(RuntimeError, match=r"torch\.no_grad\(\)"):
        tiling.decode(modules["tdec"], _x(1, 4, 2, 4, 4), tile=T3, overlap=O3)


def test_valid_calls_get_past_validation(modules):
    """Under no_grad a valid call passes every check and stops at the device (there is no CPU path)."""
    import tiling

    with torch.no_grad():
        for fn, mod, x, tile, overlap in [("encode", "tenc", _x(1, 3, 4, 8, 8), T3, O3),
                                          ("decode", "tdec", _x(1, 4, 2, 4, 4), T3, O3),
                                          ("encode", "aenc", _x(1, 3, 8, 8), (4, 4), (2, 2)),
                                          ("decode", "adec", _x(1, 4, 4, 4), (4, 4), (0, 2))]:
            with pytest.raises(RuntimeError, match="CUDA tensors only"):
                getattr(tiling, fn)(modules[mod], x, tile=tile, overlap=overlap)


def test_factors(modules):
    import ae
    import tiling

    assert [tiling.factor(modules[k]) for k in ("tenc", "tdec", "aenc", "adec")] == [2, 2, 2, 2]
    hr = ae.VAE(32, 3, 32, 3, [1, 2], 1, 4, False, True, True)
    assert tiling.factor(hr.encoder) == 2 and tiling.factor(hr.decoder) == 4


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


GOOD = dict(tile_bf16=0, N=2, C=3, T=5, H=9, W=12, Lt=2, Lh=4, Lw=8, t0=1, h0=3, w0=4, pt=1, ph=5, pw=4, nt=2, nh=9,
            nw=12)
BAD_ABI = [
    ("tile null", {"null": "tile"}),
    ("acc null", {"null": "acc"}),
    ("wt null", {"null": "wt"}),
    ("wh null", {"null": "wh"}),
    ("ww null", {"null": "ww"}),
    ("tile_bf16 = 2", {"tile_bf16": 2}),
    ("tile_bf16 < 0", {"tile_bf16": -1}),
    ("N = 0", {"N": 0}),
    ("C = 0", {"C": 0}),
    ("T = 0", {"T": 0}),
    ("W < 0", {"W": -4}),
    ("Lt = 0", {"Lt": 0}),
    ("Lw < 0", {"Lw": -8}),
    ("t window past T", {"t0": 4, "pt": 4, "nt": 5}),
    ("h window past H", {"Lh": 7, "nh": 9}),
    ("w window past W", {"w0": 5, "pw": 5}),
    ("negative start", {"h0": -1, "ph": 0}),
    ("window past INT_MAX", {"W": 2 ** 31 - 1, "w0": 2 ** 31 - 4, "Lw": 8, "pw": 2 ** 31 - 4, "nw": 2 ** 31 - 1}),
    ("prev_end before window", {"pt": 0}),
    ("prev_end past window", {"ph": 8}),
    ("next_start before window", {"nw": 3}),
    ("next_start past extent", {"nt": 6}),
    ("grid too large", {"N": 2 ** 30, "C": 2 ** 30, "T": 2 ** 10, "pt": 1}),
    ("misaligned tile", {"offset": "tile"}),
    ("misaligned acc", {"offset": "acc"}),
    ("misaligned out", {"offset": "out"}),
]


def _call(L, args):
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    a = dict(GOOD)
    a.update({k: v for k, v in args.items() if k not in ("null", "offset")})
    ptrs = {k: (None if args.get("null") == k else p + (1 if args.get("offset") == k else 0))
            for k in ("tile", "acc", "out", "wt", "wh", "ww")}
    return L.vqb_tile_blend(ptrs["tile"], a["tile_bf16"], ptrs["acc"], ptrs["out"], a["N"], a["C"], a["T"], a["H"],
                            a["W"], a["Lt"], a["Lh"], a["Lw"], a["t0"], a["h0"], a["w0"], ptrs["wt"], ptrs["wh"],
                            ptrs["ww"], a["pt"], a["ph"], a["pw"], a["nt"], a["nh"], a["nw"], None)


@pytest.mark.parametrize("what, args", BAD_ABI, ids=[b[0] for b in BAD_ABI])
def test_abi_rejects_bad_arguments(lib, what, args):
    rc = _call(lib, args)
    err = lib.vqb_last_error()
    assert rc == EINVAL, (what, rc, err)
    assert b"vqb_tile_blend" in err, err


@pytest.mark.parametrize("args", [{}, {"tile_bf16": 1}, {"null": "out"}, {"w0": 3, "pw": 3, "nw": 11},
                                  {"T": 1, "Lt": 1, "t0": 0, "pt": 0, "nt": 1}])
def test_abi_without_device_is_enodevice(lib, no_device, args):
    rc = _call(lib, args)
    err = lib.vqb_last_error()
    assert rc == ENODEVICE, (rc, err)
    assert b"vqb_tile_blend" in err and b"sm_90" in err, err


# ---------------------------------------------------------------------------------------------------- compile
def test_tile_blend_compiles_without_spills(tmp_path):
    import build_native

    if not os.path.exists(build_native.NVCC):
        pytest.skip("nvcc is not installed")
    src = os.path.join(build_native.CSRC, "tiling.cu")
    r = subprocess.run([build_native.NVCC, *build_native.FLAGS, "-c", src, "-o", str(tmp_path / "tiling.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w*tile_blend_kernel\w*)'", r.stderr)
    assert len(kernels) == 4, r.stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == 4 and all(p == ("0", "0", "0") for p in props), r.stderr
