"""Host-side tile rules of the weight-gradient GEMM: ops.choose_ksplit sizes split-K from the CTA tiles
csrc/wgrad_gemm.cu launches: 128 Cout rows x ops._wgrad_tile_blocks column blocks of ops._wgrad_block_n columns
(256 columns when taps * C64 divides by 256). test_host_logic.py counts 128-column blocks; this file counts the tiles."""
import native
import ops
import plans

# the 3x3 weight-gradient shapes of the FLUX config at B=32: N, H, W, C, Cout, tile columns, CTA tiles
FLUX_WGRAD = [(32, 32, 32, 512, 512, 256, 72), (32, 256, 256, 128, 128, 128, 9), (32, 64, 64, 512, 512, 256, 72),
              (32, 128, 128, 256, 256, 256, 18), (32, 128, 128, 128, 256, 128, 18), (32, 128, 128, 512, 256, 256, 36),
              (32, 256, 256, 256, 128, 256, 9)]


def test_wgrad_column_tile_divides_the_columns():
    L = native.load()
    for taps in (1, 2, 4, 9, 16):
        for C in (8, 16, 64, 72, 128, 192, 256, 320, 512):
            cols = L.vqb_wgrad_cols(taps, C)
            assert cols == taps * ((C + 63) // 64) * 64
            bn = ops._wgrad_block_n(cols) * ops._wgrad_tile_blocks(cols)
            assert bn in (64, 128, 256) and cols % bn == 0
            assert bn == 256 or cols % (2 * bn) != 0, "the widest tile that divides the columns"


def test_ksplit_fills_waves_with_the_cta_tiles_the_kernel_launches():
    """Split-K is sized so that (CTA tiles x splits) fills ONE wave of the 132 persistent CTAs of an H100 SXM to >= 90 %
    whenever some split count can, and otherwise fills whole waves to >= 80 %, for the weight-gradient shapes of the
    FLUX config at B=32."""
    sms = ops._num_sms()
    assert ops.H100_SMS == 132
    for (N, H, W, C, Co, bn, tiles) in FLUX_WGRAD:
        g = plans.geom_s1(N, H, W, C, 3)
        cols = native.load().vqb_wgrad_cols(len(g.taps), C)
        assert ops._wgrad_block_n(cols) * ops._wgrad_tile_blocks(cols) == bn
        assert -(-Co // 128) * (cols // bn) == tiles
        ks = ops.choose_ksplit(g, Co)
        units = tiles * ks
        if any(0.9 * sms <= tiles * k <= sms for k in range(1, sms + 1)):
            assert units <= sms and units >= 0.9 * sms, (N, H, W, C, Co, ks)
        assert units >= 0.8 * sms * -(-units // sms), (N, H, W, C, Co, ks)
