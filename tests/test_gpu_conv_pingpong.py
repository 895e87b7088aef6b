"""The ping-pong schedule of the wgmma conv kernel (csrc/conv_gemm.cu): each consumer warpgroup owns every other tile of
its CTA, skips the other warpgroup's K-chunks in the shared TMA ring and starts a tile only after the other warpgroup has
passed the last ring wait of the previous tile. The fp64 element-wise bound, the guard bands and the run-twice bit
equality of test_gpu_kernel_bounds.py run at shapes that give every CTA exactly one tile (the second warpgroup idles),
one or two tiles, or three or four, with K-chunk counts below the stage count, not a multiple of it, and at least
twice it; tile counts follow the device's SM count. A slip in the ring's stage or phase bookkeeping shows as wrong data
in the one-launch-versus-per-image comparison."""
import pytest
import torch

import test_gpu_kernel_bounds as KB
import test_gpu_tae_train_bounds as TB
from test_gpu_kernel_bounds import DEV, Guarded, K, check_bits, check_stores, ok, poisoned, rnd, stream, strided_index
from test_gpu_kernel_bounds import lib  # noqa: F401  (module fixture: loads the library, skips without an sm_90 device)

pytestmark = pytest.mark.gpu

H, W = 8, 16  # one 128-pixel tile per image: bw = 16, bh = 8, bn = 1
LAYOUTS = ("1/cta", "1-2/cta", "3-4/cta")  # CTA tiles per SM
EPIS = ("", "bias", "bias+res", "stats+bias", "bias+res+stats", "relu", "mask")
BN_COUT = {16: 16, 32: 24, 64: 64, 128: 128}


def images(layout, Cout):
    """Images of H x W for the layout's tile count on this device's SMs (CTAs = min(tiles, SMs))."""
    S = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {"1/cta": S, "1-2/cta": S + S // 2 + 1, "3-4/cta": 3 * S + S // 2}[layout]
    n_tiles = -(-Cout // 128) if Cout > 64 else 1
    return max(1, tiles // n_tiles)


def bounds_and_bits(kind, shp, C, Cout, epi, store):
    KB.test_conv_gemm_bounds(kind, shp, C, Cout, epi, store)
    if "stats" in epi:  # the bounds test runs statistics launches once: the stored outputs are deterministic too
        c = KB.build_conv2d(kind, shp, C, Cout, epi, store)
        check_bits(f"conv {kind} {shp} C={C} Cout={Cout} {epi} {store}", c.launch()[0].bits(), c.launch()[0].bits())


def epilogue_cases():
    cases, k = [], 0
    for bn, cout in BN_COUT.items():
        for epi in EPIS:
            for store in ("nhwc", "nchw32"):
                if "stats" in epi and (store != "nhwc" or cout % 64):
                    continue
                cases.append((LAYOUTS[k % 3], cout, epi, store))
                k += 1
    return cases


@pytest.mark.parametrize("layout,Cout,epi,store", epilogue_cases(), ids=lambda v: str(v) if v != "" else "plain")
def test_pingpong_epilogues(layout, Cout, epi, store):
    """Every epilogue at every BLOCK_N (3x3, C = 64: 9 K-chunks, not a multiple of the 6 or 8 stages)."""
    bounds_and_bits("s1", (images(layout, Cout), H, W), 64, Cout, epi, store)


K_CASES = [("p1", 64), ("p1", 128), ("s1", 128), ("s1", 512)]  # 1, 2, 18 and 72 K-chunks


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("kind,C", K_CASES)
@pytest.mark.parametrize("Cout", (128, 40))  # BLOCK_N 128 (6 stages) and 64 (8 stages, ragged columns)
def test_pingpong_k_chunks(layout, kind, C, Cout):
    epi, store = ("bias+res+stats", "nhwc") if Cout == 128 else ("bias+res", "nchw32" if C == 128 else "nhwc")
    bounds_and_bits(kind, (images(layout, Cout), H, W), C, Cout, epi, store)


@pytest.mark.parametrize("shp,C,Cout,epi", [((16, 64, 64), 64, 128, "stats+bias"),
                                            ((12, 32, 32), 128, 256, "bias+res+stats")])
def test_pingpong_statistics_across_warpgroups(shp, C, Cout, epi):
    """32 or 8 tiles per image over 3-4 tiles per CTA: the tiles of one image land on both warpgroups."""
    bounds_and_bits("s1", shp, C, Cout, epi, "nhwc")


@pytest.mark.parametrize("kind,C,Cout", [("p1", 64, 64), ("s1", 128, 136), ("s1", 512, 128)])
def test_one_launch_matches_per_image_launches(kind, C, Cout):
    """bias + residual + ReLU over N images in one launch (3-4 tiles per CTA) stores the same bits as N launches of
    one image each (every tile on warpgroup 0 of its CTA)."""
    P, L = K.plans, K.L
    N = images("3-4/cta", Cout)
    gen = torch.Generator(device=DEV).manual_seed(C + Cout)
    Cs, Cso, k = C + 8, P.cpad(Cout), 1 if kind == "p1" else 3
    A = poisoned(rnd(N, H, W, C, gen=gen), Cs)
    Wg = poisoned(rnd(Cout, k * k * C, scale=(k * k * C) ** -0.5, gen=gen), k * k * C)
    bias = Guarded(Cout, torch.float32, poison="nan")
    bias.body.copy_(torch.randn(Cout, device=DEV, generator=gen))
    res = Guarded(N * H * W * Cso, torch.bfloat16, poison="nan")
    res.body.copy_(rnd(N * H * W * Cso, gen=gen))
    strides = P.nhwc_strides(H, W, Cso)
    flags = K.native.EPI_BIAS | K.native.EPI_RES | K.native.EPI_RELU

    def desc(n):
        g = P.geom_s1(n, H, W, Cs, k)
        g.C = C
        return P.conv_desc(g, Cout, strides, flags)

    def run(d, a_off, o_off, out):
        ok(L.vqb_conv_gemm(d, A.ptr(a_off), Wg.ptr(), bias.ptr(), res.ptr(o_off), 0, out.ptr(o_off), 0, stream()),
           f"conv_gemm {kind}")

    whole = Guarded(N * H * W * Cso, torch.bfloat16)
    run(desc(N), 0, 0, whole)
    single = Guarded(N * H * W * Cso, torch.bfloat16)
    d1 = desc(1)
    for n in range(N):
        run(d1, n * H * W * Cs, n * H * W * Cso, single)
    torch.cuda.synchronize()
    check_stores(whole, strided_index(0, (N, H, W, Cout), strides), f"conv {kind} C={C} Cout={Cout} N={N} stores")
    same = torch.equal(whole.bits(), single.bits())
    print(f"  conv {kind} C={C} Cout={Cout}: one launch of {N} images == {N} one-image launches: {same}", flush=True)
    assert same, f"conv {kind} C={C} Cout={Cout}: one launch over {N} images differs from per-image launches"


def test_pingpong_conv3d():
    """27 taps x 2 K-chunks (54 >= 2 x 6 stages), 512 tiles: 3-4 per CTA."""
    KB.test_conv3d_gemm_bounds("s1", (2, 16, 32, 32), 72, 256, "bias+res", "nthwc")


def test_pingpong_conv3d_dgrad_64_taps():
    """64 taps x 2 K-chunks, 384 tiles: 2-3 per CTA."""
    TB.test_up_dgrad_64_taps_bounds((3, 8, 32, 32), 72, 256)
