// Convolution weight gradient on Hopper wgmma tensor cores.
//
//   dWp[co][t*C64 + c] = sum_{n,h,w} dy[n,h,w,co] * X_view(t)[n, h+dh_t, w+dw_t, c]
//
// GEMM view: M = Cout (tiles of 128, two consumer warpgroups of 64 rows), N = ntaps*C64 flattened (tap, channel)
// columns in wgmma blocks of BLOCK_N = 128 or 64 (a whole number of 64-channel atoms), K = output pixels walked in
// boxes of 64 pixels. A CTA tile is NB column blocks wide: two 128-column blocks when the columns divide by 256 (the
// tile may then span two taps), else one. Both operands stream from L2, so the tile width sets the bytes moved per
// FLOP: 16 KB dy + 16 KB x per K block at 128 columns, 16 KB + 32 KB for twice the work at 256 (a quarter less). Two
// blocks are 128 accumulator registers per consumer thread: the warpgroups re-split the register file at the role
// split (setmaxnreg: producer 40, consumers 232).
// Both operands are "MN-major": dy[pixel][co] and x[pixel][c] have the GEMM M/N index contiguous and K (the pixel)
// strided, which wgmma consumes directly (transposed operands) from 128B-swizzled [64 px][64 ch] atoms (no transposes,
// no im2col buffer). The tap shift is a coordinate offset of the TMA box and conv padding is TMA zero fill. K is split
// across CTAs (ksplit); each split writes its fp32 partial tile with plain vector stores, vqb_wgrad_reduce sums the
// splits deterministically and emits the OIHW fp32 gradient the optimizer sees.
//
// Replaces the wgrad half of aten::convolution_backward for the trainable convs of ae.py and the
// PatchDiscriminator (reference call sites listed in include/vqb200.h).
#include "common.cuh"
#include "ptx.cuh"

#include <cstring>

namespace vqb {

constexpr int kWM = 128;       // Cout rows per tile
constexpr int kWThreads = 384;  // warpgroup 0: TMA producer; warpgroups 1, 2: 64 Cout rows each
constexpr int kWMaxStages = 8;
constexpr int kWPix = 64;                     // pixels per K block
constexpr uint32_t kAtomBytes = kWPix * 128;  // [64 px][64 ch] bf16
constexpr int kWProducerRegs = 40, kWConsumerRegs = 232;

// wgmma column block and blocks per CTA tile for `cols` (tap, channel) columns; ops._wgrad_block_n and
// ops._wgrad_tile_blocks mirror them to size split-K.
static int wgrad_block_n(int cols) { return cols % 128 == 0 ? 128 : 64; }
static int wgrad_tile_blocks(int cols) { return cols % 256 == 0 ? 2 : 1; }

struct alignas(64) WgradParams {
    static constexpr int kRank = 4;  // NHWC, 4-D TMA boxes [64 ch][bw][bh][bn]
    CUtensorMap ymap;
    CUtensorMap xmap[VQB_MAX_VIEWS];
    int32_t tap_view[VQB_MAX_TAPS];
    int32_t tap_dw[VQB_MAX_TAPS];
    int32_t tap_dh[VQB_MAX_TAPS];
    int32_t ntaps, C, C64, Cout;
    int32_t lbw, lbh, lbn;
    int32_t tiles_w, tiles_h, pixel_boxes;
    int32_t n_tiles, ksplit, total_units;
    int32_t stages;
    int64_t ld;  // row stride of the partial buffer
    float* partial;
};

// The rank-5 (video) form: NTHWC, 5-D TMA boxes [64 ch][bw][bh][bt][bn] of 64 voxels, up to 27 taps over up to 8 views.
struct alignas(64) Wgrad3dParams {
    static constexpr int kRank = 5;
    CUtensorMap ymap;
    CUtensorMap xmap[VQB_MAX_VIEWS_3D];
    int32_t tap_view[VQB_MAX_TAPS_3D];
    int32_t tap_dw[VQB_MAX_TAPS_3D];
    int32_t tap_dh[VQB_MAX_TAPS_3D];
    int32_t tap_dt[VQB_MAX_TAPS_3D];
    int32_t ntaps, C, C64, Cout;
    int32_t lbw, lbh, lbt, lbn;
    int32_t tiles_w, tiles_h, tiles_t, pixel_boxes;
    int32_t n_tiles, ksplit, total_units;
    int32_t stages;
    int64_t ld;
    float* partial;
};

template <int BN, int NB, class P>
__global__ void __launch_bounds__(kWThreads, 1) wgrad_gemm_kernel(const __grid_constant__ P p) {
    extern __shared__ uint8_t smem_raw[];
    constexpr int kAtoms = NB * BN / 64;
    constexpr uint32_t kABytes = 2 * kAtomBytes;
    constexpr uint32_t kStageBytes = kABytes + kAtoms * kAtomBytes;
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const uint32_t stages = p.stages;
    uint64_t* full = reinterpret_cast<uint64_t*>(base + stages * kStageBytes);
    uint64_t* empty = full + stages;
    const uint32_t wg = threadIdx.x >> 7;
    const uint32_t warp = (threadIdx.x >> 5) & 3u;
    const uint32_t lane = threadIdx.x & 31u;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.ymap);
        tma_prefetch_desc(&p.xmap[0]);
        for (uint32_t i = 0; i < stages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8);  // lane 0 of every consumer warp releases the stage
        }
        fence_mbar_init();
    }
    __syncthreads();

    // unit -> (m_tile, n_tile, split); splits of one tile are adjacent so they share L2-resident x/dy
    auto unit_range = [&](int unit, int& m_tile, int& n_tile, int& s, int& kb0, int& kb1) {
        s = unit % p.ksplit;
        const int tile = unit / p.ksplit;
        n_tile = tile % p.n_tiles;
        m_tile = tile / p.n_tiles;
        kb0 = static_cast<int>((static_cast<int64_t>(p.pixel_boxes) * s) / p.ksplit);
        kb1 = static_cast<int>((static_cast<int64_t>(p.pixel_boxes) * (s + 1)) / p.ksplit);
    };

    if (wg == 0) {
        // ===================== TMA producer (one elected thread) =====================
        setmaxnreg_dec<kWProducerRegs>();
        if (warp == 0 && elect_one()) {
            uint32_t stage = 0, phase = 0;
            for (int unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
                int m_tile, n_tile, s, kb0, kb1;
                unit_range(unit, m_tile, n_tile, s, kb0, kb1);
                const int co0 = m_tile * kWM;
                const int colbase = n_tile * (NB * BN);
                // CTAs working on the same pixel split stream the same x / dy boxes in lock-step, so each box is
                // fetched from HBM once and hit in L2 by the other tiles
                for (int kb = kb0; kb < kb1; ++kb) {
                    const int tw = kb % p.tiles_w;
                    const int th = (kb / p.tiles_w) % p.tiles_h;
                    int tt = 0, tn;
                    if constexpr (P::kRank == 5) {
                        tt = (kb / (p.tiles_w * p.tiles_h)) % p.tiles_t;
                        tn = kb / (p.tiles_w * p.tiles_h * p.tiles_t);
                    } else {
                        tn = kb / (p.tiles_w * p.tiles_h);
                    }
                    const int w0 = tw << p.lbw, h0 = th << p.lbh, n0 = tn << p.lbn;
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full[stage], kStageBytes);
                    uint8_t* a = base + stage * kStageBytes;
                    uint8_t* b = a + kABytes;
                    if constexpr (P::kRank == 5) {
                        const int t0 = tt << p.lbt;
                        tma_load_5d(&p.ymap, &full[stage], a, co0, w0, h0, t0, n0);
                        tma_load_5d(&p.ymap, &full[stage], a + kAtomBytes, co0 + 64, w0, h0, t0, n0);
#pragma unroll
                        for (int j = 0; j < kAtoms; ++j) {
                            const int col = colbase + 64 * j;
                            const int t = col / p.C64;
                            const int c0 = col - t * p.C64;
                            tma_load_5d(&p.xmap[p.tap_view[t]], &full[stage], b + j * kAtomBytes, c0, w0 + p.tap_dw[t],
                                        h0 + p.tap_dh[t], t0 + p.tap_dt[t], n0);
                        }
                    } else {
                        tma_load_4d(&p.ymap, &full[stage], a, co0, w0, h0, n0);
                        tma_load_4d(&p.ymap, &full[stage], a + kAtomBytes, co0 + 64, w0, h0, n0);
#pragma unroll
                        for (int j = 0; j < kAtoms; ++j) {
                            const int col = colbase + 64 * j;
                            const int t = col / p.C64;
                            const int c0 = col - t * p.C64;
                            tma_load_4d(&p.xmap[p.tap_view[t]], &full[stage], b + j * kAtomBytes, c0, w0 + p.tap_dw[t],
                                        h0 + p.tap_dh[t], n0);
                        }
                    }
                    if (++stage == stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cw owns Cout rows 64*cw .. 64*cw + 63 of every tile =====================
    setmaxnreg_inc<kWConsumerRegs>();
    const uint32_t cw = wg - 1;
    const uint32_t ring = smem_u32(base);
    float acc[NB][BN / 2];  // acc[nb]: columns BN*nb .. BN*nb + BN - 1 of the tile
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[nb][i] = 0.f;
    uint32_t stage = 0, phase = 0;
    for (int unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
        int m_tile, n_tile, s, kb0, kb1;
        unit_range(unit, m_tile, n_tile, s, kb0, kb1);
        uint32_t prev = 0;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint32_t a = ring + stage * kStageBytes;
            // MN-major, 128B swizzle: SBO = 8 K-rows (1024 B), LBO = next 64-wide MN atom
            const uint64_t da = make_smem_desc(a + cw * kAtomBytes, kAtomBytes, 1024);
            const uint64_t db = make_smem_desc(a + kABytes, kAtomBytes, 1024);
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) fence_operands(acc[nb]);
            wgmma_fence();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb)  // the block's first atom (descriptor addresses count 16 B)
#pragma unroll
                for (int k = 0; k < kWPix / 16; ++k)  // 16 pixel rows of 128 B per K = 16 step
                    wgmma_bf16<BN, 1, 1>(acc[nb], da + 128 * k, db + nb * (BN / 64) * (kAtomBytes >> 4) + 128 * k,
                                         (kb > kb0 || k > 0) ? 1u : 0u);
            wgmma_commit();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) fence_operands(acc[nb]);
            // keep this K-block's group in flight while the next stage is awaited; the previous one has retired
            wgmma_wait<1>();
            if (kb > kb0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = stage;
            if (++stage == stages) {
                stage = 0;
                phase ^= 1;
            }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) fence_operands(acc[nb]);  // the epilogue's reads of acc stay below the wait
        if (kb1 > kb0 && lane == 0) mbar_arrive(&empty[prev]);
        // ---------------- epilogue: fp32 partial tile -> global
        const bool empty_range = (kb1 <= kb0);  // more splits than pixel boxes: contributes zeros
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int co = m_tile * kWM + static_cast<int>(cw * 64 + warp * 16 + (lane >> 2)) + 8 * i;
            if (co >= p.Cout) continue;
            float* orow = p.partial + (static_cast<int64_t>(s) * p.Cout + co) * p.ld + n_tile * (NB * BN) +
                          2 * (lane & 3u);
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const float2 f = empty_range ? make_float2(0.f, 0.f)
                                                 : make_float2(acc[nb][4 * j + 2 * i], acc[nb][4 * j + 2 * i + 1]);
                    *reinterpret_cast<float2*>(orow + nb * BN + 8 * j) = f;
                }
            }
        }
    }
}

template <int BN, int NB, class P>
static int launch_wgrad(const P& p, void* stream) {
    const size_t smem = 1024 + static_cast<size_t>(p.stages) * (2 + NB * BN / 64) * kAtomBytes + 16 * p.stages;
    static bool attr_set = false;
    if (!attr_set) {
        VQB_CUDA(cudaFuncSetAttribute(wgrad_gemm_kernel<BN, NB, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    const int grid = p.total_units < num_sms() ? p.total_units : num_sms();
    wgrad_gemm_kernel<BN, NB, P><<<grid, kWThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
    VQB_CUDA(cudaGetLastError());
    return VQB_OK;
}

template <class P>
static int launch_wgrad_form(int block_n, int tile_n, const P& p, void* stream) {
    if (tile_n == 256) return launch_wgrad<128, 2>(p, stream);
    return block_n == 128 ? launch_wgrad<128, 1>(p, stream) : launch_wgrad<64, 1>(p, stream);
}

static int encode_view(const VqbView& vw, const void* basep, int C, int lbw, int lbh, int lbn, CUtensorMap* m) {
    const void* base = static_cast<const uint8_t*>(basep) + vw.offset * 2;
    uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(vw.Wv), static_cast<uint64_t>(vw.Hv),
                        static_cast<uint64_t>(vw.Nv)};
    uint64_t str[3] = {static_cast<uint64_t>(vw.sw) * 2, static_cast<uint64_t>(vw.sh) * 2,
                       static_cast<uint64_t>(vw.sn) * 2};
    uint32_t box[4] = {64, 1u << lbw, 1u << lbh, 1u << lbn};
    return encode_tmap_bf16(m, base, 4, dims, str, box, 128);
}

}  // namespace vqb

using namespace vqb;

extern "C" int vqb_wgrad_cols(int ntaps, int C) { return ntaps * ((C + 63) / 64) * 64; }

extern "C" int vqb_wgrad_gemm(const VqbWgradDesc* d, const void* dy, const void* x, float* partial, void* stream) {
    VQB_CHECK(d && dy && x && partial, "vqb_wgrad_gemm: null pointer");
    VQB_CHECK(d->C > 0 && d->C % 8 == 0 && d->Cout > 0 && d->Cout % 8 == 0,
              "vqb_wgrad_gemm: C=%d Cout=%d must be positive multiples of 8", d->C, d->Cout);
    VQB_CHECK(d->ntaps >= 1 && d->ntaps <= VQB_MAX_TAPS && d->nviews >= 1 && d->nviews <= VQB_MAX_VIEWS,
              "vqb_wgrad_gemm: ntaps/nviews out of range");
    VQB_CHECK(d->ksplit >= 1, "vqb_wgrad_gemm: ksplit must be >= 1");
    VQB_CHECK((reinterpret_cast<uintptr_t>(partial) & 15u) == 0, "vqb_wgrad_gemm: partial not 16-byte aligned");
    VQB_CHECK(d->col_offset % 2 == 0 && d->ld_override % 2 == 0,
              "vqb_wgrad_gemm: col_offset / ld_override must be even (8-byte partial stores)");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_wgrad_gemm: current device is not sm_90");

    WgradParams p;
    const uint32_t kp = kWPix;
    uint32_t bw = next_pow2(d->W);
    if (bw > kp) bw = kp;
    uint32_t bh = next_pow2(d->H);
    if (bh > kp / bw) bh = kp / bw;
    uint32_t bn = kp / (bw * bh);
    p.lbw = ilog2(bw);
    p.lbh = ilog2(bh);
    p.lbn = ilog2(bn);
    p.tiles_w = (d->W + bw - 1) / bw;
    p.tiles_h = (d->H + bh - 1) / bh;
    p.pixel_boxes = p.tiles_w * p.tiles_h * ((d->N + bn - 1) / bn);
    p.ntaps = d->ntaps;
    p.C = d->C;
    p.C64 = ((d->C + 63) / 64) * 64;
    p.Cout = d->Cout;
    const int cols = vqb_wgrad_cols(d->ntaps, d->C);
    const int block_n = wgrad_block_n(cols), tile_n = block_n * wgrad_tile_blocks(cols);
    const int m_tiles = (d->Cout + kWM - 1) / kWM;
    p.n_tiles = cols / tile_n;
    p.ksplit = d->ksplit;
    p.total_units = m_tiles * p.n_tiles * p.ksplit;
    // ld_override / col_offset: several launches may fill column ranges of one partial buffer (folded upsample conv)
    p.ld = d->ld_override > 0 ? d->ld_override : cols;
    p.partial = partial + d->col_offset;
    const int stage_bytes = (2 + tile_n / 64) * static_cast<int>(kAtomBytes);
    int stages = (200 * 1024) / stage_bytes;
    if (stages > kWMaxStages) stages = kWMaxStages;
    p.stages = stages;
    for (int t = 0; t < d->ntaps; ++t) {
        VQB_CHECK(d->taps[t].view >= 0 && d->taps[t].view < d->nviews, "vqb_wgrad_gemm: tap view out of range");
        p.tap_view[t] = d->taps[t].view;
        p.tap_dw[t] = d->taps[t].dw;
        p.tap_dh[t] = d->taps[t].dh;
    }
    int rc = encode_view(d->dy_view, dy, d->Cout, p.lbw, p.lbh, p.lbn, &p.ymap);
    if (rc != VQB_OK) return rc;
    for (int v = 0; v < d->nviews; ++v) {
        rc = encode_view(d->views[v], x, d->C, p.lbw, p.lbh, p.lbn, &p.xmap[v]);
        if (rc != VQB_OK) return rc;
    }
    rc = launch_wgrad_form(block_n, tile_n, p, stream);
    if (rc != VQB_OK) return rc;
    count_launch();
    return VQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Rank-5 weight gradient of the video autoencoder's 3x3x3 convs (tae.py call sites in include/vqb200.h).
static int encode_view3d(const VqbView3d& vw, const void* basep, int C, uint32_t bw, uint32_t bh, uint32_t bt,
                         uint32_t bn, CUtensorMap* m) {
    const void* base = static_cast<const uint8_t*>(basep) + vw.offset * 2;
    uint64_t dims[5] = {static_cast<uint64_t>(C), static_cast<uint64_t>(vw.Wv), static_cast<uint64_t>(vw.Hv),
                        static_cast<uint64_t>(vw.Tv), static_cast<uint64_t>(vw.Nv)};
    uint64_t str[4] = {static_cast<uint64_t>(vw.sw) * 2, static_cast<uint64_t>(vw.sh) * 2,
                       static_cast<uint64_t>(vw.st) * 2, static_cast<uint64_t>(vw.sn) * 2};
    uint32_t box[5] = {64, bw, bh, bt, bn};
    return vqb::encode_tmap_bf16(m, base, 5, dims, str, box, 128);
}

static bool view3d_ok(const VqbView3d& vw) {
    return vw.offset >= 0 && vw.Wv > 0 && vw.Hv > 0 && vw.Tv > 0 && vw.Nv > 0 && vw.sw > 0 && vw.sw % 8 == 0 &&
           vw.sh > 0 && vw.sh % 8 == 0 && vw.st > 0 && vw.st % 8 == 0 && vw.sn > 0 && vw.sn % 8 == 0;
}

extern "C" int vqb_wgrad3d_gemm(const VqbWgrad3dDesc* d, const void* dy, const void* x, float* partial, void* stream) {
    VQB_CHECK(d && dy && x && partial, "vqb_wgrad3d_gemm: null pointer");
    VQB_CHECK(d->C > 0 && d->C % 8 == 0 && d->Cout > 0 && d->Cout % 8 == 0,
              "vqb_wgrad3d_gemm: C=%d Cout=%d must be positive multiples of 8", d->C, d->Cout);
    VQB_CHECK(d->N > 0 && d->T > 0 && d->H > 0 && d->W > 0, "vqb_wgrad3d_gemm: bad extents");
    VQB_CHECK(d->ntaps >= 1 && d->ntaps <= VQB_MAX_TAPS_3D && d->nviews >= 1 && d->nviews <= VQB_MAX_VIEWS_3D,
              "vqb_wgrad3d_gemm: ntaps=%d nviews=%d out of range", d->ntaps, d->nviews);
    VQB_CHECK(d->ksplit >= 1, "vqb_wgrad3d_gemm: ksplit must be >= 1");
    VQB_CHECK((reinterpret_cast<uintptr_t>(partial) & 15u) == 0, "vqb_wgrad3d_gemm: partial not 16-byte aligned");
    VQB_CHECK(d->col_offset >= 0 && d->ld_override >= 0 && d->col_offset % 2 == 0 && d->ld_override % 2 == 0,
              "vqb_wgrad3d_gemm: col_offset / ld_override must be non-negative and even (8-byte partial stores)");
    VQB_CHECK(view3d_ok(d->dy_view), "vqb_wgrad3d_gemm: dy view has bad extents / strides");
    for (int v = 0; v < d->nviews; ++v)
        VQB_CHECK(view3d_ok(d->views[v]), "vqb_wgrad3d_gemm: view %d has bad extents / strides", v);
    for (int t = 0; t < d->ntaps; ++t)
        VQB_CHECK(d->taps[t].view >= 0 && d->taps[t].view < d->nviews, "vqb_wgrad3d_gemm: tap %d view out of range",
                  t);
    const int cols = vqb_wgrad_cols(d->ntaps, d->C);
    if (d->ld_override > 0)
        VQB_CHECK(d->col_offset + cols <= d->ld_override, "vqb_wgrad3d_gemm: columns exceed ld_override");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_wgrad3d_gemm: current device is not sm_90");

    Wgrad3dParams p;
    memset(&p, 0, sizeof(p));
    // 64-voxel K box: as wide as the video (<= 64), then as tall, then as deep, then across videos
    const uint32_t kp = kWPix;
    uint32_t bw = next_pow2(d->W);
    if (bw > kp) bw = kp;
    uint32_t bh = next_pow2(d->H);
    if (bh > kp / bw) bh = kp / bw;
    uint32_t bt = next_pow2(d->T);
    if (bt > kp / (bw * bh)) bt = kp / (bw * bh);
    const uint32_t bn = kp / (bw * bh * bt);
    p.lbw = ilog2(bw);
    p.lbh = ilog2(bh);
    p.lbt = ilog2(bt);
    p.lbn = ilog2(bn);
    p.tiles_w = (d->W + bw - 1) / bw;
    p.tiles_h = (d->H + bh - 1) / bh;
    p.tiles_t = (d->T + bt - 1) / bt;
    const int64_t boxes = static_cast<int64_t>(p.tiles_w) * p.tiles_h * p.tiles_t * ((d->N + bn - 1) / bn);
    VQB_CHECK(boxes < (1ll << 31), "vqb_wgrad3d_gemm: too many voxel boxes");
    p.pixel_boxes = static_cast<int32_t>(boxes);
    p.ntaps = d->ntaps;
    p.C = d->C;
    p.C64 = ((d->C + 63) / 64) * 64;
    p.Cout = d->Cout;
    const int block_n = wgrad_block_n(cols), tile_n = block_n * wgrad_tile_blocks(cols);
    const int m_tiles = (d->Cout + kWM - 1) / kWM;
    p.n_tiles = cols / tile_n;
    p.ksplit = d->ksplit;
    const int64_t units = static_cast<int64_t>(m_tiles) * p.n_tiles * p.ksplit;
    VQB_CHECK(units < (1ll << 31), "vqb_wgrad3d_gemm: too many work units");
    p.total_units = static_cast<int32_t>(units);
    p.ld = d->ld_override > 0 ? d->ld_override : cols;
    p.partial = partial + d->col_offset;
    const int stage_bytes = (2 + tile_n / 64) * static_cast<int>(kAtomBytes);
    int stages = (200 * 1024) / stage_bytes;
    if (stages > kWMaxStages) stages = kWMaxStages;
    p.stages = stages;
    for (int t = 0; t < d->ntaps; ++t) {
        p.tap_view[t] = d->taps[t].view;
        p.tap_dw[t] = d->taps[t].dw;
        p.tap_dh[t] = d->taps[t].dh;
        p.tap_dt[t] = d->taps[t].dt;
    }
    int rc = encode_view3d(d->dy_view, dy, d->Cout, bw, bh, bt, bn, &p.ymap);
    if (rc != VQB_OK) return rc;
    for (int v = 0; v < d->nviews; ++v) {
        rc = encode_view3d(d->views[v], x, d->C, bw, bh, bt, bn, &p.xmap[v]);
        if (rc != VQB_OK) return rc;
    }
    rc = launch_wgrad_form(block_n, tile_n, p, stream);
    if (rc != VQB_OK) return rc;
    count_launch();
    return VQB_OK;
}
