"""GPU (-m gpu): tiled encode / decode (tiling.py, csrc/tiling.cu; DESIGN.md section 3.11, section 7 row 27).

Bound. The kernel computes p = (wt * wh) * ww from fp32 tables and accumulates acc = p * v, then
acc = fmaf(p, v, acc) for each further tile covering the element. Against the float64 blend with the unrounded float64
weights, every element is off by at most gamma_m * S with S = sum over the covering tiles of |w v| and m = 3 table
roundings + 2 products + one rounding per contributing tile (k, up to 12 here), gamma_m = m u / (1 - m u), u = 2^-24.
A bf16 output adds its one rounding: |out - ref| <= gamma_m S (1 + 2^-8) + 2^-8 |ref|. The tile values are exact in float64, so nothing else enters.

Kernel cases launch vqb_tile_blend directly into NaN-sentinel buffers with 4 KB guard bands over a grid larger than the
plan: every element the plan covers is written, and the guard bands and every element outside the plan keep their
sentinel bits. Module cases run tiling.encode / tiling.decode on TVAE SMALL (f = 2) and small ae.VAEs (plain, HR
decoder, wavelet encoder) in fp32 and bf16, and check the result against the float64 blend of the module's own outputs
on each window (recomputed; the no-grad forward is deterministic, which the test checks). Reruns are bit-identical.

`python -m pytest -m gpu -q tests/test_gpu_tiling.py -s` prints max(err/bound) per case.
"""
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import seeded
from oracle import tae_oracle as TAO
from oracle import tiling_oracle as TO
from test_gpu_kernel_bounds import Guarded, check_stores, worst

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
U_BF16 = 2.0 ** -8
SMALL = TAO.TAEConfig(ch=32, ch_mult=(1, 8), num_res_blocks=1, z_channels=4, resolution=16)


@pytest.fixture(scope="module", autouse=True)
def lib():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import native

    L = native.load()
    if not L.vqb_device_ok():
        pytest.skip("needs an sm_90 device")
    return L


def gamma(m):
    return m * U / (1 - m * U)


def counts(axes):
    """Contributing tiles per element of the grid, [*gextent] float64."""
    c = np.ones(())
    for a in axes:
        n = np.zeros(a["gextent"])
        for s in a["gstarts"]:
            n[s:s + a["glen"]] += 1
        c = np.multiply.outer(c, n)
    return c


def bound(axes, tiles, ref, bf16_out):
    S = TO.blend({k: np.abs(v) for k, v in tiles.items()}, axes)
    b = gamma(5 + counts(axes)) * S
    if bf16_out:
        b = b * (1 + U_BF16) + U_BF16 * np.abs(ref)
    return b


def check(name, got, ref, b):
    r, info = worst(got, torch.from_numpy(ref).cuda(), torch.from_numpy(b).cuda())
    print(f"  {name}: max(err/bound)={r:.3g}  {info}", flush=True)
    assert r <= 1.0, f"{name}: max(err/bound)={r:.3g}, {info}"


# ---------------------------------------------------------------------------------------------------- the kernel
# (name, N, C, latent extents (T, H, W), tile, overlap, f, decode, tile dtype, bf16 output)
KERNEL_CASES = [
    ("ragged W tails, C=3, T=1", 1, 3, (1, 9, 13), (4, 32, 32), (0, 16, 16), 4, False, torch.float32, False),
    ("unaligned latent windows, C=32", 2, 32, (5, 7, 23), (4, 6, 8), (2, 2, 4), 2, False, torch.float32, False),
    ("bf16 tiles, bf16 output", 1, 3, (6, 10, 18), (4, 8, 8), (2, 4, 4), 2, True, torch.bfloat16, True),
    ("bf16 tiles, C=32, latent grid", 1, 32, (4, 11, 37), (2, 6, 10), (0, 2, 4), 2, False, torch.bfloat16, True),
    ("uneven plan, overlaps wider than R", 1, 3, (7, 23, 41), (4, 8, 12), (2, 2, 4), 1, True, torch.float32, False),
    ("fp32 tiles, bf16 output, vector path", 1, 32, (3, 12, 16), (16, 32, 32), (8, 8, 16), 8, True, torch.float32,
     True),
]
PAD = (1, 2, 4)  # the plan sits at this origin of a grid PAD larger on both sides (W: keeps 4-aligned rows possible)


def run_kernel_case(c, seed):
    import native
    import tiling

    name, N, C, X, tile, overlap, f, decode, dt, bf16_out = c
    axes = [TO.axis(Xa, L, O, f, decode) for Xa, L, O in zip(X, tile, overlap)]
    tables = [tiling._Axis(Xa, L, O, f, decode).table.cuda() for Xa, L, O in zip(X, tile, overlap)]
    ext = [a["gextent"] + 2 * p for a, p in zip(axes, PAD)]
    gen = torch.Generator(device="cuda").manual_seed(seed)
    tiles = {idx: torch.randn(N, C, *(a["glen"] for a in axes), device="cuda", generator=gen).to(dt)
             for idx in itertools.product(*(range(len(a["gstarts"])) for a in axes))}
    acc = Guarded(N * C * math.prod(ext), torch.float32)
    out = Guarded(N * C * math.prod(ext), torch.bfloat16) if bf16_out else None
    L = native.load()
    for idx, y in tiles.items():
        o = [a["gstarts"][k] + p for a, k, p in zip(axes, idx, PAD)]
        pe = [(a["gstarts"][k - 1] + a["glen"] if k > 0 else a["gstarts"][k]) + p for a, k, p in zip(axes, idx, PAD)]
        ns = [(a["gstarts"][k + 1] if k < len(a["gstarts"]) - 1 else a["gextent"]) + p
              for a, k, p in zip(axes, idx, PAD)]
        native.check(L.vqb_tile_blend(y.data_ptr(), int(dt == torch.bfloat16), acc.ptr(), out.ptr() if out else None,
                                      N, C, *ext, *(a["glen"] for a in axes), *o,
                                      *(t[k].data_ptr() for t, k in zip(tables, idx)), *pe, *ns,
                                      native.stream_ptr()), name)
    torch.cuda.synchronize()
    return axes, ext, tiles, acc, out


@pytest.mark.parametrize("case", KERNEL_CASES, ids=[c[0] for c in KERNEL_CASES])
def test_kernel_against_float64(case):
    name, N, C = case[:3]
    bf16_out = case[-1]
    axes, ext, tiles, acc, out = run_kernel_case(case, 0)
    t64 = {k: v.double().cpu().numpy() for k, v in tiles.items()}
    ref = TO.blend(t64, axes)
    inner = (slice(None), slice(None)) + tuple(slice(p, p + a["gextent"]) for a, p in zip(axes, PAD))
    idx = torch.arange(N * C * math.prod(ext), device="cuda").view(N, C, *ext)[inner]
    b = bound(axes, t64, ref, False)
    check(f"{name} (fp32 acc)", acc.body.view(N, C, *ext)[inner], ref, b)
    check_stores(acc, idx, f"{name} (acc)")
    if bf16_out:
        check(f"{name} (bf16 out)", out.body.view(N, C, *ext)[inner], ref, bound(axes, t64, ref, True))
        check_stores(out, idx, f"{name} (bf16 out)")
    _, _, _, acc2, out2 = run_kernel_case(case, 0)
    assert torch.equal(acc.bits(), acc2.bits()), f"{name}: reruns differ"
    if bf16_out:
        assert torch.equal(out.bits(), out2.bits()), f"{name}: reruns differ (bf16 out)"


def test_bound_rejects_a_wrong_weight():
    """The checker bites: the blend with one tile's T weight table shifted by one entry is rejected."""
    case = KERNEL_CASES[2]
    name, N, C = case[:3]
    axes, ext, tiles, acc, _ = run_kernel_case(case, 1)
    t64 = {k: v.double().cpu().numpy() for k, v in tiles.items()}
    ref = TO.blend(t64, axes)
    bad = [dict(a) for a in axes]
    bad[0]["weights"] = np.roll(axes[0]["weights"], 1, axis=1)
    inner = (slice(None), slice(None)) + tuple(slice(p, p + a["gextent"]) for a, p in zip(axes, PAD))
    r, _ = worst(acc.body.view(N, C, *ext)[inner], torch.from_numpy(TO.blend(t64, bad)).cuda(),
                 torch.from_numpy(bound(axes, t64, ref, False)).cuda())
    assert r > 1.0, "a shifted weight table was accepted"


# ---------------------------------------------------------------------------------------------------- modules
def tvae(dtype):
    import tae

    m = tae.TVAE(**SMALL.kwargs())
    m.load_state_dict(seeded.fill_state_dict(m.state_dict(), "tiling/tvae"))
    return m.cuda().to(dtype).eval()


def ae_vae(dtype, hr=False, wavelet=False):
    import ae

    m = ae.VAE(32, 3, 32, 3, [1, 2], 1, 4, False, hr, wavelet)
    m.load_state_dict(seeded.fill_state_dict(m.state_dict(), f"tiling/ae/{hr}/{wavelet}"))
    return m.cuda().to(dtype).eval()


def module_cases():
    """(name, make module, which part, input shape, tile, overlap)"""
    cases = []
    for dt in (torch.float32, torch.bfloat16):
        d = "fp32" if dt == torch.float32 else "bf16"
        cases += [
            (f"tvae encode {d}", lambda dt=dt: tvae(dt).encoder, False, (1, 3, 8, 32, 48), (4, 16, 16), (2, 4, 4)),
            (f"tvae decode {d}", lambda dt=dt: tvae(dt).decoder, True, (1, 4, 4, 16, 24), (4, 16, 16), (2, 4, 4)),
            (f"ae encode {d}", lambda dt=dt: ae_vae(dt).encoder, False, (2, 3, 64, 96), (32, 32), (8, 8)),
            (f"ae decode {d}", lambda dt=dt: ae_vae(dt).decoder, True, (2, 4, 32, 48), (32, 32), (8, 8)),
            (f"ae hr decode {d}", lambda dt=dt: ae_vae(dt, hr=True).decoder, True, (1, 4, 24, 40), (32, 48),
             (8, 16)),
            (f"ae wavelet encode {d}", lambda dt=dt: ae_vae(dt, wavelet=True).encoder, False, (1, 3, 64, 80),
             (32, 32), (8, 16)),
        ]
    return cases


MODULE_CASES = module_cases()


def _input(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g).clamp(-1, 1)


@pytest.mark.parametrize("case", MODULE_CASES, ids=[c[0] for c in MODULE_CASES])
def test_module_tiled_equals_the_blend_of_its_windows(case):
    import tiling

    name, make, decode, shape, tile, overlap = case
    m = make()
    f = tiling.factor(m)
    x = _input(shape, 3)
    with torch.no_grad():
        got = (tiling.decode if decode else tiling.encode)(m, x, tile=tile, overlap=overlap)
        again = (tiling.decode if decode else tiling.encode)(m, x, tile=tile, overlap=overlap)
        assert torch.equal(got, again), f"{name}: tiled reruns differ"
        X = shape[2:] if decode else tuple(e // f for e in shape[2:])
        axes = [TO.axis(Xa, L, O, f, decode) for Xa, L, O in zip(X, tile, overlap)]
        assert any(len(a["gstarts"]) > 1 for a in axes)
        s = 1 if decode else f
        tiles = {}
        for idx in itertools.product(*(range(len(a["gstarts"])) for a in axes)):
            win = tuple(slice(a["starts"][k] * s, (a["starts"][k] + a["length"]) * s) for a, k in zip(axes, idx))
            y = m(x[(slice(None), slice(None)) + win].contiguous())
            assert torch.equal(y, m(x[(slice(None), slice(None)) + win].contiguous())), f"{name}: forward varies"
            tiles[idx] = y.double().cpu().numpy()
    dt = next(m.parameters()).dtype
    assert got.dtype == dt and tuple(got.shape) == tuple(next(iter(tiles.values())).shape[:2]) + tuple(
        a["gextent"] for a in axes)
    ref = TO.blend(tiles, axes)
    check(name, got, ref, bound(axes, tiles, ref, dt == torch.bfloat16))


@pytest.mark.parametrize("case", MODULE_CASES, ids=[c[0] for c in MODULE_CASES])
def test_one_tile_is_the_module_itself(case):
    import native
    import tiling

    name, make, decode, shape, _, _ = case
    m = make()
    f = tiling.factor(m)
    x = _input(shape, 4)
    tile = tuple(e * f if decode else e for e in shape[2:])
    with torch.no_grad():
        m(x)  # packs the weights once, so that both counts below are of forwards alone
        n0 = native.launch_count()
        want = m(x)
        n1 = native.launch_count()
        got = (tiling.decode if decode else tiling.encode)(m, x, tile=tile, overlap=(0,) * len(tile))
        n2 = native.launch_count()
    assert torch.equal(got, want), f"{name}: one tile differs from module(x)"
    assert n2 - n1 == n1 - n0, f"{name}: {n2 - n1} launches against the module's {n1 - n0}"


# ---------------------------------------------------------------------------------------------------- memory
def test_decode_memory_follows_the_tile_not_the_clip():
    import tae
    import tiling

    cfg = TAO.TAEConfig(ch=64, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=16, resolution=256)
    m = tae.TVAE(**cfg.kwargs())
    m.load_state_dict(seeded.fill_state_dict(m.state_dict(), "tiling/mem"))
    dec = m.decoder.cuda().eval()
    tile, overlap = (16, 256, 256), (8, 64, 64)
    peaks, outs = {}, {}
    with torch.no_grad():
        for frames in (16, 48, 16, 48):  # the first two warm up
            z = _input((1, 16, frames // 8, 32, 32), frames)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            y = tiling.decode(dec, z, tile=tile, overlap=overlap)
            torch.cuda.synchronize()
            peaks[frames] = torch.cuda.max_memory_allocated() - base
            outs[frames] = y.numel() * y.element_size()
            del y
        z = _input((1, 16, 6, 32, 32), 48)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        y = dec(z)
        torch.cuda.synchronize()
        untiled = torch.cuda.max_memory_allocated() - base
        del y
    growth, allowed = peaks[48] - peaks[16], outs[48] - outs[16] + 64 * 2 ** 20  # fp32 decoder: acc is the output
    print(f"  peak 16 frames {peaks[16] / 2**20:.1f} MiB, 48 frames {peaks[48] / 2**20:.1f} MiB tiled, "
          f"{untiled / 2**20:.1f} MiB untiled; growth {growth / 2**20:.1f} MiB (allowed {allowed / 2**20:.1f})")
    assert growth <= allowed
    assert peaks[48] < untiled
