// Implicit-GEMM convolution on Hopper wgmma tensor cores (forward and data-gradient).
//
//   out[n,h,w,co] = epi( sum_t sum_c A_view(t)[n, h+dh_t, w+dw_t, c] * Wp[co][t*C + c] )
//
// GEMM view: M = output pixels (tiles of 128 = BW x BH x BN box of the NHWC tensor), N = Cout (tiles of BLOCK_N),
// K = ntaps * C walked in 64-channel chunks. Per K-chunk the TMA producer issues ONE 4-D tiled load of the activation
// box shifted by the tap offset (out-of-range rows/cols/channels are zero-filled by the TMA unit -> conv padding costs
// nothing) and ONE 2-D load of the packed weights; both land in 128B-swizzled K-major smem tiles of a multi-stage
// mbarrier ring. Persistent: one CTA per SM walks tiles round-robin, and its two consumer warpgroups take turns
// ("ping-pong"): warpgroup c owns the CTA's tiles of local index = c (mod 2) whole, issuing two wgmma row blocks
// (M = 64 each, N = BLOCK_N, K = 16 x4) per K-chunk into 2 x BLOCK_N / 2 fp32 accumulators per thread, so one
// warpgroup's epilogue (bias / residual / ReLU / mask / GroupNorm statistics -> bf16 NHWC or strided fp32) runs while
// the other warpgroup's MMAs run. 128 accumulators per thread at BLOCK_N = 128 need the register file re-split at the
// role split (setmaxnreg: producer 40, consumers 232).
//
// Math order: a warpgroup starts the K loop of its tile only after the other warpgroup has passed the last `full`
// wait of the previous tile (the `order` mbarriers). The ring's full barriers are waited by parity alone, so without
// this a warpgroup two or more fills behind on a stage would take the other warpgroup's chunk for its own; with it,
// every full barrier a consumer waits on has completed all earlier fills, for any K-chunk count and stage count.
//
// Staged epilogue (kStaged; NHWC bf16 outputs, Cout % 64 == 0, short K: the rule is in conv_gemm_impl): each consumer
// warpgroup owns a 128 x BLOCK_N bf16 tile buffer after the ring, BLOCK_N / 64 slabs of [128 rows][128 B] in the ring's
// 128B swizzle, guarded by epi_full[c] / epi_empty[c] (count 1 each). Tile l of a CTA belongs to warpgroup c = l & 1 and
// is the (l >> 1)-th use of its buffer; both barriers are waited with parity (l >> 1) & 1, epi_empty with the ring's
// "previous phase" convention (the first wait passes).
//   producer, before tile l's K-chunks: wait epi_empty[c], then TMA-load the tile's residual or mask box into the buffer
//     (complete_tx on epi_full[c]), or arrive on epi_full[c] when there is none. The load lands during the MMAs.
//   warpgroup c, after its MMAs: wait epi_full[c]; each thread reads its residual / mask and writes the rounded bf16
//     result in the same place (generic proxy), fence.proxy.async.shared::cta, 128-thread named barrier; one thread
//     issues one TMA store per slab, commits, and after the statistics waits cp.async.bulk.wait_group.read 0 (the
//     buffer has been read) before it arrives on epi_empty[c]. It waits for full completion before the CTA exits.
// So the buffer is written by TMA only after the previous tile's store has read it, and by the threads only after that
// load (or the producer's plain arrival, which itself followed the read) completed.
//
// Replaces the cuDNN kernels behind nn.Conv2d at reference ae.py:105-117,143-154,160-167 and the
// torchvision VGG convs reached from utils.py:95-111,150-154 (see include/vqb200.h).
#include "common.cuh"
#include "ptx.cuh"

#include <cstring>

namespace vqb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KB per stage
constexpr int kThreads = 384;                   // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue
constexpr int kMaxStages = 8;
constexpr int kConsumerWarps = 8;
constexpr int kProducerRegs = 40;   // setmaxnreg split: 40 * 128 + 232 * 256 <= 64 K registers
constexpr int kConsumerRegs = 232;
constexpr int kStagedKChunksPerTensor = 18;  // staged-epilogue rule in conv_gemm_impl (DESIGN.md 3.1)

struct alignas(64) ConvParams {
    static constexpr int kRank = 4;  // NHWC activations, 4-D TMA boxes [64 ch][bw][bh][bn]
    static constexpr int kViews = VQB_MAX_VIEWS;
    CUtensorMap amap[VQB_MAX_VIEWS];
    CUtensorMap bmap;
    CUtensorMap omap;  // staged epilogue: the output as [Cout][W][H][N], box [64 ch][bw][bh][bn]
    CUtensorMap emap;  // staged epilogue: the residual or the mask, same extents, strides and box as omap
    int32_t tap_view[VQB_MAX_TAPS];
    int32_t tap_dw[VQB_MAX_TAPS];
    int32_t tap_dh[VQB_MAX_TAPS];
    int32_t ntaps, kchunks, C, Cout;
    int32_t N, H, W;
    int32_t lbw, lbh, lbn;
    int32_t tiles_w, tiles_h;
    int32_t n_tiles, total_tiles;
    int32_t stages, do_stats;
    int32_t flags, out_f32;
    int32_t vec_store, _pad0;  // 1: paired bf16 stores (oc == 1, 16-byte aligned pixel rows), else per element
    int64_t on, oh, ow, oc;
    void* out;
    const void* res;
    const void* mask;
    const float* bias;
    float* stats;
};

// The 3-D (video) form: NTHWC activations, 5-D TMA boxes [64 ch][bw][bh][bt][bn], up to 27 taps over up to 8 views.
// The epilogue has bias and residual; the statistics / ReLU / mask fields exist so that the kernel
// body compiles for both ranks, and are always zero here (the kernel tests kRank before reading them). kTaps is the size
// of the tap table: 27 (vqb_conv3d_gemm) or 64 (vqb_conv3d_dgrad_gemm, the data gradient of the folded up-sampling).
template <int kTaps>
struct alignas(64) Conv3dParamsT {
    static constexpr int kRank = 5;
    static constexpr int kViews = VQB_MAX_VIEWS_3D;
    CUtensorMap amap[VQB_MAX_VIEWS_3D];
    CUtensorMap bmap;
    int32_t tap_view[kTaps];
    int32_t tap_dw[kTaps];
    int32_t tap_dh[kTaps];
    int32_t tap_dt[kTaps];
    int32_t ntaps, kchunks, C, Cout;
    int32_t N, T, H, W;
    int32_t lbw, lbh, lbt, lbn;
    int32_t tiles_w, tiles_h, tiles_t;
    int32_t n_tiles, total_tiles;
    int32_t stages, do_stats;
    int32_t flags, out_f32;
    int32_t vec_store, _pad0;
    int64_t on, ot, oh, ow, oc;
    void* out;
    const void* res;
    const void* mask;
    const float* bias;
    float* stats;
};
using Conv3dParams = Conv3dParamsT<VQB_MAX_TAPS_3D>;
using Conv3dDgradParams = Conv3dParamsT<VQB_MAX_TAPS_3D_DGRAD>;

template <int BN, class P, bool kStaged>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_kernel(const __grid_constant__ P p) {
    constexpr bool kR5 = P::kRank == 5;
    static_assert(!kStaged || (!kR5 && BN >= 64), "the staged epilogue stores whole 64-channel slabs of 2-D outputs");
    extern __shared__ uint8_t smem_raw[];
    constexpr uint32_t kBBytes = BN * kBlockK * 2;
    constexpr uint32_t kStageBytes = kABytes + kBBytes;  // a multiple of 2 KB: every tile stays 1024-B aligned
    // carve shared memory (1024-B aligned for the 128B swizzle atoms)
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const uint32_t stages = p.stages;
    // staged epilogue: one 128 x BN bf16 tile per consumer warpgroup, as BN / 64 slabs of [128 rows][64 ch] in the
    // ring's 128B swizzle (what a [64 ch][bw][bh][bn] TMA box writes), after the ring
    constexpr uint32_t kSlabBytes = kBlockM * kBlockK * 2;
    constexpr uint32_t kEpiBytes = kBlockM * BN * 2;
    constexpr uint32_t kRowOff[4] = {0, 8 * 128, 64 * 128, 72 * 128};  // row groups r = 2 mb + i: rows + 64 mb + 8 i
    uint8_t* epi = base + stages * kStageBytes;
    float* sStat = reinterpret_cast<float*>(epi + (kStaged ? 2 * kEpiBytes : 0));  // [2 warpgroups][4 warps][BN][2]
    uint64_t* full = reinterpret_cast<uint64_t*>(sStat + kConsumerWarps * BN * 2);
    uint64_t* empty = full + stages;
    uint64_t* order = empty + stages;  // [warpgroup]: one phase per tile, completed at its last full wait
    uint64_t* epi_full = order + 2;    // [warpgroup]: its tile buffer holds the residual / mask (or is free to write)
    uint64_t* epi_empty = epi_full + 2;  // [warpgroup]: the TMA store of its previous tile has read the buffer
    const uint32_t wg = threadIdx.x >> 7;
    const uint32_t warp = (threadIdx.x >> 5) & 3u;  // warp inside its warpgroup
    const uint32_t lane = threadIdx.x & 31u;

    if (threadIdx.x == 0) {
        for (int v = 0; v < P::kViews; ++v) {
            bool used = false;
            for (int t = 0; t < p.ntaps; ++t) used |= (p.tap_view[t] == v);
            if (used) tma_prefetch_desc(&p.amap[v]);
        }
        tma_prefetch_desc(&p.bmap);
        if constexpr (kStaged) {
            tma_prefetch_desc(&p.omap);
            if (p.flags & (VQB_EPI_RES | VQB_EPI_MASK)) tma_prefetch_desc(&p.emap);
        }
        for (uint32_t i = 0; i < stages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 4);  // lane 0 of every warp of the consuming warpgroup releases the stage
        }
        for (int c = 0; c < 2; ++c) {
            mbar_init(&order[c], 4);
            mbar_init(&epi_full[c], 1);
            mbar_init(&epi_empty[c], 1);
        }
        fence_mbar_init();
    }
    __syncthreads();

    const int num_kb = p.ntaps * p.kchunks;
    if (wg == 0) {
        // ===================== TMA producer (one elected thread), tiles in order =====================
        setmaxnreg_dec<kProducerRegs>();
        if (warp == 0 && elect_one()) {
            uint32_t stage = 0, phase = 0;
            for (int tile = blockIdx.x, l = 0; tile < p.total_tiles; tile += gridDim.x, ++l) {
                const int n_tile = tile % p.n_tiles;
                const int m_tile = tile / p.n_tiles;
                const int tw = m_tile % p.tiles_w;
                const int th = (m_tile / p.tiles_w) % p.tiles_h;
                int tt = 0, tn;
                if constexpr (kR5) {
                    tt = (m_tile / (p.tiles_w * p.tiles_h)) % p.tiles_t;
                    tn = m_tile / (p.tiles_w * p.tiles_h * p.tiles_t);
                } else {
                    tn = m_tile / (p.tiles_w * p.tiles_h);
                }
                const int w0 = tw << p.lbw, h0 = th << p.lbh, n0 = tn << p.lbn;
                const int ncol0 = n_tile * BN;
                if constexpr (kStaged) {
                    // tile l goes to warpgroup l & 1: once its buffer is free (the store of tile l - 2 has read
                    // it), fill it with this tile's residual or mask; it lands while the tile's MMAs run
                    const uint32_t c = l & 1;
                    mbar_wait(&epi_empty[c], ((l >> 1) & 1) ^ 1);
                    if (p.flags & (VQB_EPI_RES | VQB_EPI_MASK)) {
                        const int nslab = min(BN, p.Cout - ncol0) / kBlockK;  // Cout % 64 == 0
                        mbar_arrive_expect_tx(&epi_full[c], nslab * kSlabBytes);
                        for (int s = 0; s < nslab; ++s)
                            tma_load_4d(&p.emap, &epi_full[c], epi + c * kEpiBytes + s * kSlabBytes,
                                        ncol0 + s * kBlockK, w0, h0, n0);
                    } else {
                        mbar_arrive(&epi_full[c]);
                    }
                }
                for (int t = 0; t < p.ntaps; ++t) {
                    for (int kc = 0; kc < p.kchunks; ++kc) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        uint8_t* a_dst = base + stage * kStageBytes;
                        mbar_arrive_expect_tx(&full[stage], kStageBytes);
                        if constexpr (kR5)
                            tma_load_5d(&p.amap[p.tap_view[t]], &full[stage], a_dst, kc * kBlockK, w0 + p.tap_dw[t],
                                        h0 + p.tap_dh[t], (tt << p.lbt) + p.tap_dt[t], n0);
                        else
                            tma_load_4d(&p.amap[p.tap_view[t]], &full[stage], a_dst, kc * kBlockK, w0 + p.tap_dw[t],
                                        h0 + p.tap_dh[t], n0);
                        tma_load_2d(&p.bmap, &full[stage], a_dst + kABytes, t * p.C + kc * kBlockK, ncol0);
                        if (++stage == stages) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cw owns the CTA's tiles 2i + cw, all 128 rows of each ==============
    setmaxnreg_inc<kConsumerRegs>();
    const uint32_t cw = wg - 1;
    const uint32_t cwarp = cw * 4 + warp;  // 0..7
    const uint32_t wtid = threadIdx.x & 127u;  // thread inside its warpgroup
    const uint32_t ring = smem_u32(base);
    const bool has_bias = p.flags & VQB_EPI_BIAS, has_res = p.flags & VQB_EPI_RES;
    const bool do_relu = !kR5 && (p.flags & VQB_EPI_RELU), has_mask = !kR5 && (p.flags & VQB_EPI_MASK);
    const bool vec_path = p.vec_store != 0;
    const bool reduce = !kR5 && p.do_stats;
    const __nv_bfloat16* res = reinterpret_cast<const __nv_bfloat16*>(p.res);
    const __nv_bfloat16* mask = reinterpret_cast<const __nv_bfloat16*>(p.mask);
    float acc[2][BN / 2];  // acc[mb]: rows 64*mb .. 64*mb + 63 of the tile
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[mb][i] = 0.f;
    uint32_t stage = 0, phase = 0;
    for (int l = static_cast<int>(cw);; l += 2) {  // l: the CTA's local tile index
        const int tile = blockIdx.x + l * gridDim.x;
        if (tile >= p.total_tiles) break;
        if (l > 0) {
            // tile l - 1 is the other warpgroup's: skip its K-chunks in the ring, and start only once it has passed
            // its last full wait (phase (l - 1) / 2 of its order barrier)
            stage += num_kb;
            phase ^= (stage / stages) & 1u;
            stage %= stages;
            mbar_wait(&order[cw ^ 1u], ((l - 1) >> 1) & 1);
        }
        uint32_t prev = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&full[stage], phase);
            if (kb == num_kb - 1 && lane == 0) mbar_arrive(&order[cw]);
            const uint32_t a = ring + stage * kStageBytes;
            const uint64_t da0 = make_smem_desc(a, 16, 1024);
            const uint64_t da1 = make_smem_desc(a + 8192u, 16, 1024);  // rows 64..127: 64 rows x 128 B further
            const uint64_t db = make_smem_desc(a + kABytes, 16, 1024);
            fence_operands(acc[0]);
            fence_operands(acc[1]);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k) {  // +32 B per K = 16 step inside the swizzle atom
                wgmma_bf16<BN, 0, 0>(acc[0], da0 + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
                wgmma_bf16<BN, 0, 0>(acc[1], da1 + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            fence_operands(acc[0]);
            fence_operands(acc[1]);
            // keep this K-chunk's group in flight while the next stage is awaited; the previous one has retired
            wgmma_wait<1>();
            if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = stage;
            if (++stage == stages) {
                stage = 0;
                phase ^= 1;
            }
        }
        wgmma_wait<0>();
        fence_operands(acc[0]);  // the epilogue's reads of acc stay below the wait
        fence_operands(acc[1]);
        if (lane == 0) mbar_arrive(&empty[prev]);  // num_kb >= 1 (ntaps >= 1, C > 0)

        // ---------------- epilogue: from the accumulator fragment to global memory, or through the staged tile
        const int n_tile = tile % p.n_tiles;
        const int m_tile = tile / p.n_tiles;
        const int tw = m_tile % p.tiles_w;
        const int th = (m_tile / p.tiles_w) % p.tiles_h;
        int tt = 0, tn;
        if constexpr (kR5) {
            tt = (m_tile / (p.tiles_w * p.tiles_h)) % p.tiles_t;
            tn = m_tile / (p.tiles_w * p.tiles_h * p.tiles_t);
        } else {
            tn = m_tile / (p.tiles_w * p.tiles_h);
        }
        const int col0 = n_tile * BN;
        uint8_t* tbuf = epi + cw * kEpiBytes;  // staged: this warpgroup's tile buffer
        // staged: this thread's column pair in row group 0 (row % 8 == lane / 4 in all four row groups)
        const uint32_t trow = smem_u32(tbuf) + (warp * 16 + (lane >> 2)) * 128u + (lane & 3u) * 4u;
        if (kStaged) mbar_wait(&epi_full[cw], (l >> 1) & 1);
        // row group r = 2 * mb + i: acc[mb][4j + 2i + e] is row 64 mb + 16 warp + lane / 4 + 8 i, column 8j + 2(lane % 4) + e
        int64_t pix[4] = {0, 0, 0, 0};
        bool valid[4] = {true, true, true, true};  // staged: rows outside the tensor are computed, then clipped by TMA
        if constexpr (!kStaged) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const uint32_t row = (r >> 1) * 64 + warp * 16 + (lane >> 2) + 8 * (r & 1);  // row of the 128-pixel box
                const int w = (tw << p.lbw) + static_cast<int>(row & ((1u << p.lbw) - 1));
                const int h = (th << p.lbh) + static_cast<int>((row >> p.lbw) & ((1u << p.lbh) - 1));
                if constexpr (kR5) {  // row = w + bw * (h + bh * (t + bt * n)) of the 128-voxel box
                    const int t = (tt << p.lbt) + static_cast<int>((row >> (p.lbw + p.lbh)) & ((1u << p.lbt) - 1));
                    const int n = (tn << p.lbn) + static_cast<int>(row >> (p.lbw + p.lbh + p.lbt));
                    valid[r] = (w < p.W) && (h < p.H) && (t < p.T) && (n < p.N);
                    pix[r] = static_cast<int64_t>(n) * p.on + static_cast<int64_t>(t) * p.ot +
                             static_cast<int64_t>(h) * p.oh + static_cast<int64_t>(w) * p.ow;
                } else {
                    const int n = (tn << p.lbn) + static_cast<int>(row >> (p.lbw + p.lbh));
                    valid[r] = (w < p.W) && (h < p.H) && (n < p.N);
                    pix[r] = static_cast<int64_t>(n) * p.on + static_cast<int64_t>(h) * p.oh +
                             static_cast<int64_t>(w) * p.ow;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int col = col0 + j * 8 + 2 * static_cast<int>(lane & 3u);
            const bool ok0 = col < p.Cout, ok1 = col + 1 < p.Cout;
            float b0 = 0.f, b1 = 0.f;
            if (has_bias) {
                b0 = ok0 ? __ldg(p.bias + col) : 0.f;
                b1 = ok1 ? __ldg(p.bias + col + 1) : 0.f;
            }
            float r1[2] = {0.f, 0.f}, r2[2] = {0.f, 0.f};  // per column: statistics partial sums over this thread's rows
            if (kStaged ? ok1 : vec_path && ok1) {
                // all residual / mask loads of the column group in flight before the first use
                __nv_bfloat162 rv[4], mv[4];
                // staged: 16-byte chunk j % 8 of a 128-B row, XOR row % 8 (128B swizzle). The 8 rows a warp touches
                // per access fall in 8 different chunks, so these loads and stores are free of bank conflicts.
                const uint32_t tj = trow + (j >> 3) * kSlabBytes + (((j & 7u) ^ (lane >> 2)) << 4);
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    rv[r] = mv[r] = __floats2bfloat162_rn(0.f, 0.f);
                    if constexpr (kStaged) {
                        if (has_res || has_mask) {
                            const __nv_bfloat162 v = u32_as_bf16x2(ld_shared_u32(tj + kRowOff[r]));
                            if (has_res) rv[r] = v;
                            if (has_mask) mv[r] = v;
                        }
                        continue;
                    }
                    const int64_t o = pix[r] + col;  // 4-byte aligned: pixel strides % 8 == 0, col even
                    if (has_res && valid[r]) rv[r] = *reinterpret_cast<const __nv_bfloat162*>(res + o);
                    if (has_mask && valid[r]) mv[r] = *reinterpret_cast<const __nv_bfloat162*>(mask + o);
                }
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (!valid[r]) continue;
                    const int a0 = 4 * j + 2 * (r & 1);
                    float f[2] = {acc[r >> 1][a0] + b0, acc[r >> 1][a0 + 1] + b1};
                    if (has_res) {
                        const float2 rf = __bfloat1622float2(rv[r]);
                        f[0] += rf.x;
                        f[1] += rf.y;
                    }
                    if (do_relu) {
                        f[0] = fmaxf(f[0], 0.f);
                        f[1] = fmaxf(f[1], 0.f);
                    }
                    if (has_mask) {
                        const float2 m = __bfloat1622float2(mv[r]);
                        if (!(m.x > 0.f)) f[0] = 0.f;
                        if (!(m.y > 0.f)) f[1] = 0.f;
                    }
                    const __nv_bfloat162 ob = __floats2bfloat162_rn(f[0], f[1]);
                    if constexpr (kStaged)
                        st_shared_u32(tj + kRowOff[r], bf16x2_as_u32(ob));  // in place of its residual / mask
                    else
                        *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.out) + pix[r] + col) = ob;
                    if (reduce) {
                        const float2 v = __bfloat1622float2(ob);  // the bf16 values the consumer will read
                        r1[0] += v.x;
                        r2[0] = fmaf(v.x, v.x, r2[0]);
                        r1[1] += v.y;
                        r2[1] = fmaf(v.y, v.y, r2[1]);
                    }
                }
            } else if constexpr (!kStaged) {
                // generic strided / ragged path (small or odd Cout, NCHW fp32 outputs)
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (!valid[r]) continue;
                    const int a0 = 4 * j + 2 * (r & 1);
                    const float f[2] = {acc[r >> 1][a0] + b0, acc[r >> 1][a0 + 1] + b1};
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (!(e ? ok1 : ok0)) continue;
                        const int64_t o = pix[r] + static_cast<int64_t>(col + e) * p.oc;
                        float x = f[e];
                        if (has_res) x += __bfloat162float(res[o]);
                        if (do_relu) x = fmaxf(x, 0.f);
                        if (has_mask && !(__bfloat162float(mask[o]) > 0.f)) x = 0.f;
                        if (p.out_f32)
                            reinterpret_cast<float*>(p.out)[o] = x;
                        else
                            reinterpret_cast<__nv_bfloat16*>(p.out)[o] = __float2bfloat16(x);
                    }
                }
            }
            if (reduce) {  // warp-uniform: sum the 8 row groups of the warp (lane bits 2..4), then stage per warp
#pragma unroll
                for (int off = 4; off < 32; off <<= 1) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        r1[e] += __shfl_xor_sync(0xffffffffu, r1[e], off);
                        r2[e] += __shfl_xor_sync(0xffffffffu, r2[e], off);
                    }
                }
                if (lane < 4) {
                    float* s = sStat + (cwarp * BN + j * 8 + 2 * lane) * 2;
                    *reinterpret_cast<float4*>(s) = make_float4(r1[0], r2[0], r1[1], r2[1]);
                }
            }
        }
        if constexpr (kStaged) {
            // the tile's generic-proxy writes, then one thread hands it to the TMA unit: one store per 64-channel slab
            // inside Cout (rows outside the tensor are clipped by TMA)
            fence_proxy_async_shared();
            named_bar_sync(1 + cw, 128);
            if (wtid == 0) {
                const int nslab = min(BN, p.Cout - col0) / kBlockK;
                for (int s = 0; s < nslab; ++s)
                    tma_store_4d(&p.omap, tbuf + s * kSlabBytes, col0 + s * kBlockK, tw << p.lbw, th << p.lbh,
                                 tn << p.lbn);
                bulk_commit_group();
            }
        }
        if (reduce) {
            // the statistics need every row of the tile inside one image (checked on the host: vqb_conv_stats_ok)
            named_bar_sync(1 + cw, 128);
            const int n_img = tn << p.lbn;
            const float* sw = sStat + cw * 4 * BN * 2;
            for (uint32_t idx = wtid; idx < BN * 2u; idx += 128u) {
                const int c = col0 + static_cast<int>(idx >> 1);
                float v = 0.f;
#pragma unroll
                for (int w4 = 0; w4 < 4; ++w4) v += sw[w4 * BN * 2 + idx];
                if (c < p.Cout) atomicAdd(p.stats + (static_cast<int64_t>(n_img) * p.Cout + c) * 2 + (idx & 1u), v);
            }
            named_bar_sync(1 + cw, 128);  // this warpgroup's sStat half is reused by its next tile
        }
        if (kStaged && wtid == 0) {
            bulk_wait_group_read<0>();  // the buffer is free: the producer may load tile l + 2's residual / mask
            mbar_arrive(&epi_empty[cw]);
        }
    }
    if (kStaged && wtid == 0) bulk_wait_group<0>();  // the last tile's stores are complete before the CTA exits
}

static int fill_views(const VqbView* views, int nviews, const void* a, int C, int lbw, int lbh, int lbn,
                      CUtensorMap* maps) {
    for (int v = 0; v < nviews; ++v) {
        const VqbView& vw = views[v];
        uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(vw.Wv), static_cast<uint64_t>(vw.Hv),
                            static_cast<uint64_t>(vw.Nv)};
        uint64_t str[3] = {static_cast<uint64_t>(vw.sw) * 2, static_cast<uint64_t>(vw.sh) * 2,
                           static_cast<uint64_t>(vw.sn) * 2};
        uint32_t box[4] = {kBlockK, 1u << lbw, 1u << lbh, 1u << lbn};
        const void* base = static_cast<const uint8_t*>(a) + vw.offset * 2;
        int rc = encode_tmap_bf16(&maps[v], base, 4, dims, str, box, 128);
        if (rc != VQB_OK) return rc;
    }
    return VQB_OK;
}

// Dynamic shared memory of one CTA: alignment slack, ring, the two staged epilogue tiles, statistics staging, the
// full / empty barriers of the ring and the order / epi_full / epi_empty pairs.
static size_t conv_smem_bytes(int block_n, int stages, bool staged) {
    return 1024 + static_cast<size_t>(stages) * (kABytes + block_n * kBlockK * 2) +
           (staged ? 2 * kBlockM * block_n * 2 : 0) + kConsumerWarps * block_n * 2 * sizeof(float) + 8 * (2 * stages + 6);
}

// The deepest ring (<= kMaxStages) that fits next to the rest: 6 stages at BLOCK_N = 128 and 8 below it, or 4 and 7
// when the staged epilogue tiles take their 64 / 32 KB.
static int ring_stages(int block_n, bool staged) {
    int stages = kMaxStages;
    while (conv_smem_bytes(block_n, stages, staged) > 227 * 1024) --stages;
    return stages;
}

template <int BN, bool kStaged = false, class P>
static int launch_conv(const P& p, void* stream) {
    const size_t smem = conv_smem_bytes(BN, p.stages, kStaged);
    static bool attr_set = false;
    if (!attr_set) {
        VQB_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, P, kStaged>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      227 * 1024));
        attr_set = true;
    }
    const int grid = p.total_tiles < num_sms() ? p.total_tiles : num_sms();
    conv_gemm_kernel<BN, P, kStaged><<<grid, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
    VQB_CUDA(cudaGetLastError());
    return VQB_OK;
}

}  // namespace vqb

using namespace vqb;

static int conv_gemm_impl(const VqbConvDesc* d, const void* a, const void* w_packed, const float* bias, const void* res,
                          const void* mask, void* out, float* stats, void* stream, bool query_only);

extern "C" int vqb_conv_gemm(const VqbConvDesc* d, const void* a, const void* w_packed, const float* bias,
                             const void* res, const void* mask, void* out, float* stats, void* stream) {
    return conv_gemm_impl(d, a, w_packed, bias, res, mask, out, stats, stream, false);
}

// 1 if vqb_conv_gemm can produce GroupNorm statistics (VQB_EPI_STATS) for this descriptor, else 0.
extern "C" int vqb_conv_stats_ok(const VqbConvDesc* d) {
    if (!d) return 0;
    VqbConvDesc q = *d;
    q.flags &= ~VQB_EPI_STATS;
    alignas(16) static const uint64_t dummy_aligned[4] = {0, 0, 0, 0};
    const void* dp = dummy_aligned;
    const int r = conv_gemm_impl(&q, dp, dp, static_cast<const float*>(dp), dp, dp, const_cast<void*>(dp), nullptr,
                                 nullptr, true);
    return r == 1 ? 1 : 0;
}

static int conv_gemm_impl(const VqbConvDesc* d, const void* a, const void* w_packed, const float* bias, const void* res,
                          const void* mask, void* out, float* stats, void* stream, bool query_only) {
    VQB_CHECK(d && a && w_packed && out, "vqb_conv_gemm: null pointer");
    VQB_CHECK(d->C > 0 && d->C % 8 == 0, "vqb_conv_gemm: C=%d must be a positive multiple of 8", d->C);
    VQB_CHECK(d->Cout > 0 && d->N > 0 && d->H > 0 && d->W > 0, "vqb_conv_gemm: bad extents");
    VQB_CHECK(d->ntaps >= 1 && d->ntaps <= VQB_MAX_TAPS && d->nviews >= 1 && d->nviews <= VQB_MAX_VIEWS,
              "vqb_conv_gemm: ntaps=%d nviews=%d out of range", d->ntaps, d->nviews);
    VQB_CHECK(((int64_t)d->ntaps * d->C) % 8 == 0, "vqb_conv_gemm: weight row stride must be 16-byte aligned");
    if ((d->flags & VQB_EPI_BIAS))
        VQB_CHECK(bias != nullptr && (reinterpret_cast<uintptr_t>(bias) & 15u) == 0,
                  "vqb_conv_gemm: VQB_EPI_BIAS needs a 16-byte aligned bias pointer");
    if ((d->flags & VQB_EPI_RES)) VQB_CHECK(res != nullptr, "vqb_conv_gemm: VQB_EPI_RES without res");
    if ((d->flags & VQB_EPI_MASK)) VQB_CHECK(mask != nullptr, "vqb_conv_gemm: VQB_EPI_MASK without mask");
    if ((d->flags & VQB_EPI_STATS)) VQB_CHECK(stats != nullptr, "vqb_conv_gemm: VQB_EPI_STATS without stats");
    // Paired bf16 stores need 16-byte aligned pixel rows. A channel-contiguous output without them (e.g. NCHW bf16 of
    // 1x1 images: oc = H*W = 1, on = Cout) takes the per-element store instead.
    const uintptr_t ops = reinterpret_cast<uintptr_t>(res) | reinterpret_cast<uintptr_t>(mask);
    const bool nhwc_bf16 = d->oc == 1 && !d->out_f32 && d->on % 8 == 0 && d->oh % 8 == 0 && d->ow % 8 == 0 &&
                           (reinterpret_cast<uintptr_t>(out) & 15u) == 0 && (ops & 3u) == 0;
    if (!nhwc_bf16)
        VQB_CHECK((reinterpret_cast<uintptr_t>(out) & (d->out_f32 ? 3u : 1u)) == 0 && (ops & 1u) == 0,
                  "vqb_conv_gemm: misaligned output / residual / mask");
    for (int t = 0; t < d->ntaps; ++t)
        VQB_CHECK(d->taps[t].view >= 0 && d->taps[t].view < d->nviews, "vqb_conv_gemm: tap %d view out of range", t);
    if (!query_only && !device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_conv_gemm: current device is not sm_90");

    ConvParams p;  // ~2.5 KB, filled per call, passed by value (__grid_constant__) to the kernel
    // BLOCK_N: 128 accumulator columns per warpgroup (64 fp32 registers per thread) for wide layers; narrow layers
    // round Cout up to the next wgmma width so that no tensor-core work is spent on padding beyond it.
    const int block_n = d->Cout > 64 ? 128 : (d->Cout > 32 ? 64 : (d->Cout > 16 ? 32 : 16));
    p.n_tiles = (d->Cout + block_n - 1) / block_n;
    // pixel box per CTA tile: 128 output pixels, as wide as the image (<= 128), then as tall, then across images
    uint32_t bw = next_pow2(d->W);
    if (bw > 128) bw = 128;
    uint32_t bh = next_pow2(d->H);
    if (bh > 128 / bw) bh = 128 / bw;
    const uint32_t bn = 128 / (bw * bh);
    p.lbw = ilog2(bw);
    p.lbh = ilog2(bh);
    p.lbn = ilog2(bn);
    p.tiles_w = (d->W + bw - 1) / bw;
    p.tiles_h = (d->H + bh - 1) / bh;
    const int tiles_nb = (d->N + bn - 1) / bn;
    p.total_tiles = p.tiles_w * p.tiles_h * tiles_nb * p.n_tiles;
    // GroupNorm statistics in the epilogue: NHWC bf16 output, every tile inside one image, no ragged tiles
    const bool stats_ok = nhwc_bf16 && bn == 1 && (d->W % bw == 0) && (d->H % bh == 0) && (d->Cout % 64 == 0);
    if (d->flags & VQB_EPI_STATS) {
        if (!stats_ok)
            return set_error(VQB_EINVAL, "vqb_conv_gemm: VQB_EPI_STATS unsupported for this shape (N=%d H=%d W=%d Cout=%d)",
                             d->N, d->H, d->W, d->Cout);
    }
    p.do_stats = (d->flags & VQB_EPI_STATS) ? 1 : 0;
    if (query_only) return stats_ok ? 1 : 0;
    // Staged epilogue (kernel header): whole 64-channel slabs of an NHWC bf16 output that TMA can address, and at most
    // one of residual / mask, 16-byte aligned like the output. It saves per tile in proportion to the tile-sized tensors
    // the epilogue moves (the output, and the residual or mask), and its two tile buffers cost the ring 2 of its 6
    // stages at BLOCK_N = 128 (1 of 8 at 64), a loss in proportion to the K-chunks of a tile: it is taken up to
    // kStagedKChunksPerTensor K-chunks per moved tensor. Everything else stores from the accumulator fragment.
    const bool has_res = d->flags & VQB_EPI_RES, has_mask = d->flags & VQB_EPI_MASK;
    const void* eop = has_res ? res : mask;
    const int moved = (has_res || has_mask) ? 2 : 1;
    const bool staged = nhwc_bf16 && d->Cout % 64 == 0 && d->on > 0 && d->oh > 0 && d->ow > 0 &&
                        !(has_res && has_mask) && (reinterpret_cast<uintptr_t>(eop) & 15u) == 0 &&
                        d->ntaps * ((d->C + kBlockK - 1) / kBlockK) <= kStagedKChunksPerTensor * moved;
    p.stages = ring_stages(block_n, staged);
    p.ntaps = d->ntaps;
    p.kchunks = (d->C + kBlockK - 1) / kBlockK;
    p.C = d->C;
    p.Cout = d->Cout;
    p.N = d->N;
    p.H = d->H;
    p.W = d->W;
    p.flags = d->flags;
    p.out_f32 = d->out_f32;
    p.vec_store = nhwc_bf16 ? 1 : 0;
    p._pad0 = 0;
    p.on = d->on;
    p.oh = d->oh;
    p.ow = d->ow;
    p.oc = d->oc;
    p.out = out;
    p.res = res;
    p.mask = mask;
    p.bias = bias;
    p.stats = stats;
    for (int t = 0; t < d->ntaps; ++t) {
        p.tap_view[t] = d->taps[t].view;
        p.tap_dw[t] = d->taps[t].dw;
        p.tap_dh[t] = d->taps[t].dh;
    }
    int rc = fill_views(d->views, d->nviews, a, d->C, p.lbw, p.lbh, p.lbn, p.amap);
    if (rc != VQB_OK) return rc;
    if (staged) {
        // the output (and the residual / mask, which share its strides) as 4-D tensors [Cout][W][H][N] in the
        // activations' box: out-of-range rows are zero-filled on load and clipped on store
        uint64_t dims[4] = {static_cast<uint64_t>(d->Cout), static_cast<uint64_t>(d->W), static_cast<uint64_t>(d->H),
                            static_cast<uint64_t>(d->N)};
        uint64_t str[3] = {static_cast<uint64_t>(d->ow) * 2, static_cast<uint64_t>(d->oh) * 2,
                           static_cast<uint64_t>(d->on) * 2};
        uint32_t box[4] = {kBlockK, bw, bh, bn};
        rc = encode_tmap_bf16(&p.omap, out, 4, dims, str, box, 128);
        if (rc == VQB_OK && (has_res || has_mask)) rc = encode_tmap_bf16(&p.emap, eop, 4, dims, str, box, 128);
        if (rc != VQB_OK) return rc;
    }
    {
        const uint64_t ktot = static_cast<uint64_t>(d->ntaps) * d->C;
        uint64_t dims[2] = {ktot, static_cast<uint64_t>(d->Cout)};
        uint64_t str[1] = {ktot * 2};
        uint32_t box[2] = {kBlockK, static_cast<uint32_t>(block_n)};
        rc = encode_tmap_bf16(&p.bmap, w_packed, 2, dims, str, box, 128);
        if (rc != VQB_OK) return rc;
    }
    switch (block_n) {
        case 16: rc = launch_conv<16>(p, stream); break;
        case 32: rc = launch_conv<32>(p, stream); break;
        case 64: rc = staged ? launch_conv<64, true>(p, stream) : launch_conv<64>(p, stream); break;
        default: rc = staged ? launch_conv<128, true>(p, stream) : launch_conv<128>(p, stream); break;
    }
    if (rc != VQB_OK) return rc;
    count_launch();
    return VQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// 3-D (video) convolution: the same kernel over NTHWC activations with 5-D TMA boxes (tae.py call sites in vqb200.h).
// D / P: VqbConv3dDesc / Conv3dParams (27 taps) or VqbConv3dDgradDesc / Conv3dDgradParams (64 taps); `fn` names the
// entry point in error messages.
template <class D, class P, int kMaxTaps>
static int conv3d_impl(const char* fn, const D* d, const void* a, const void* w_packed, const float* bias,
                       const void* res, void* out, void* stream) {
    VQB_CHECK(d && a && w_packed && out, "%s: null pointer", fn);
    VQB_CHECK(d->C > 0 && d->C % 8 == 0, "%s: C=%d must be a positive multiple of 8", fn, d->C);
    VQB_CHECK(d->Cout > 0 && d->N > 0 && d->T > 0 && d->H > 0 && d->W > 0, "%s: bad extents", fn);
    VQB_CHECK(d->ntaps >= 1 && d->ntaps <= kMaxTaps && d->nviews >= 1 && d->nviews <= VQB_MAX_VIEWS_3D,
              "%s: ntaps=%d nviews=%d out of range", fn, d->ntaps, d->nviews);
    VQB_CHECK((d->flags & ~(VQB_EPI_BIAS | VQB_EPI_RES)) == 0,
              "%s: flags 0x%x: only VQB_EPI_BIAS and VQB_EPI_RES are supported", fn, d->flags);
    VQB_CHECK(d->out_f32 == 0 || d->out_f32 == 1, "%s: out_f32 must be 0 or 1", fn);
    if (d->flags & VQB_EPI_BIAS)
        VQB_CHECK(bias != nullptr && (reinterpret_cast<uintptr_t>(bias) & 15u) == 0,
                  "%s: VQB_EPI_BIAS needs a 16-byte aligned bias pointer", fn);
    if (d->flags & VQB_EPI_RES) VQB_CHECK(res != nullptr, "%s: VQB_EPI_RES without res", fn);
    VQB_CHECK(d->on >= 0 && d->ot >= 0 && d->oh >= 0 && d->ow >= 0 && d->oc > 0,
              "%s: output strides must be non-negative (oc > 0)", fn);
    // paired bf16 stores need 16-byte aligned voxel rows; otherwise (e.g. NCTHW bf16 of 1x1x1 videos: oc = 1) the
    // per-element store
    const bool vec3 = d->oc == 1 && !d->out_f32 && d->on % 8 == 0 && d->ot % 8 == 0 && d->oh % 8 == 0 &&
                      d->ow % 8 == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0 &&
                      (reinterpret_cast<uintptr_t>(res) & 3u) == 0;
    if (!vec3)
        VQB_CHECK((reinterpret_cast<uintptr_t>(out) & (d->out_f32 ? 3u : 1u)) == 0 &&
                      (reinterpret_cast<uintptr_t>(res) & 1u) == 0,
                  "%s: misaligned output / residual", fn);
    for (int v = 0; v < d->nviews; ++v) {
        const VqbView3d& vw = d->views[v];
        VQB_CHECK(vw.offset >= 0 && vw.Wv > 0 && vw.Hv > 0 && vw.Tv > 0 && vw.Nv > 0 && vw.sw > 0 && vw.sw % 8 == 0 &&
                      vw.sh > 0 && vw.sh % 8 == 0 && vw.st > 0 && vw.st % 8 == 0 && vw.sn > 0 && vw.sn % 8 == 0,
                  "%s: view %d has bad extents / strides (strides must be positive multiples of 8)", fn, v);
    }
    for (int t = 0; t < d->ntaps; ++t)
        VQB_CHECK(d->taps[t].view >= 0 && d->taps[t].view < d->nviews, "%s: tap %d view out of range", fn, t);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "%s: current device is not sm_90", fn);

    P p;
    memset(&p, 0, sizeof(p));  // statistics / mask fields stay zero (rank-5 epilogue: bias + residual)
    const int block_n = d->Cout > 64 ? 128 : (d->Cout > 32 ? 64 : (d->Cout > 16 ? 32 : 16));
    p.n_tiles = (d->Cout + block_n - 1) / block_n;
    // voxel box per CTA tile: 128 output voxels, as wide as the video (<= 128), then as tall, then as deep, then across
    // videos
    uint32_t bw = next_pow2(d->W);
    if (bw > 128) bw = 128;
    uint32_t bh = next_pow2(d->H);
    if (bh > 128 / bw) bh = 128 / bw;
    uint32_t bt = next_pow2(d->T);
    if (bt > 128 / (bw * bh)) bt = 128 / (bw * bh);
    const uint32_t bn = 128 / (bw * bh * bt);
    p.lbw = ilog2(bw);
    p.lbh = ilog2(bh);
    p.lbt = ilog2(bt);
    p.lbn = ilog2(bn);
    p.tiles_w = (d->W + bw - 1) / bw;
    p.tiles_h = (d->H + bh - 1) / bh;
    p.tiles_t = (d->T + bt - 1) / bt;
    const int64_t total = static_cast<int64_t>(p.tiles_w) * p.tiles_h * p.tiles_t * ((d->N + bn - 1) / bn) * p.n_tiles;
    VQB_CHECK(total < (1ll << 31), "%s: too many tiles", fn);
    p.total_tiles = static_cast<int32_t>(total);
    p.stages = ring_stages(block_n, false);
    p.ntaps = d->ntaps;
    p.kchunks = (d->C + kBlockK - 1) / kBlockK;
    p.C = d->C;
    p.Cout = d->Cout;
    p.N = d->N;
    p.T = d->T;
    p.H = d->H;
    p.W = d->W;
    p.flags = d->flags;
    p.out_f32 = d->out_f32;
    p.vec_store = vec3 ? 1 : 0;
    p.on = d->on;
    p.ot = d->ot;
    p.oh = d->oh;
    p.ow = d->ow;
    p.oc = d->oc;
    p.out = out;
    p.res = res;
    p.bias = bias;
    for (int t = 0; t < d->ntaps; ++t) {
        p.tap_view[t] = d->taps[t].view;
        p.tap_dw[t] = d->taps[t].dw;
        p.tap_dh[t] = d->taps[t].dh;
        p.tap_dt[t] = d->taps[t].dt;
    }
    for (int v = 0; v < d->nviews; ++v) {
        const VqbView3d& vw = d->views[v];
        uint64_t dims[5] = {static_cast<uint64_t>(d->C), static_cast<uint64_t>(vw.Wv), static_cast<uint64_t>(vw.Hv),
                            static_cast<uint64_t>(vw.Tv), static_cast<uint64_t>(vw.Nv)};
        uint64_t str[4] = {static_cast<uint64_t>(vw.sw) * 2, static_cast<uint64_t>(vw.sh) * 2,
                           static_cast<uint64_t>(vw.st) * 2, static_cast<uint64_t>(vw.sn) * 2};
        uint32_t box[5] = {kBlockK, bw, bh, bt, bn};
        const void* vbase = static_cast<const uint8_t*>(a) + vw.offset * 2;
        int rc = encode_tmap_bf16(&p.amap[v], vbase, 5, dims, str, box, 128);
        if (rc != VQB_OK) return rc;
    }
    int rc;
    {
        const uint64_t ktot = static_cast<uint64_t>(d->ntaps) * d->C;
        uint64_t dims[2] = {ktot, static_cast<uint64_t>(d->Cout)};
        uint64_t str[1] = {ktot * 2};
        uint32_t box[2] = {kBlockK, static_cast<uint32_t>(block_n)};
        rc = encode_tmap_bf16(&p.bmap, w_packed, 2, dims, str, box, 128);
        if (rc != VQB_OK) return rc;
    }
    switch (block_n) {
        case 16: rc = launch_conv<16>(p, stream); break;
        case 32: rc = launch_conv<32>(p, stream); break;
        case 64: rc = launch_conv<64>(p, stream); break;
        default: rc = launch_conv<128>(p, stream); break;
    }
    if (rc != VQB_OK) return rc;
    count_launch();
    return VQB_OK;
}

extern "C" int vqb_conv3d_gemm(const VqbConv3dDesc* d, const void* a, const void* w_packed, const float* bias,
                               const void* res, void* out, void* stream) {
    return conv3d_impl<VqbConv3dDesc, Conv3dParams, VQB_MAX_TAPS_3D>("vqb_conv3d_gemm", d, a, w_packed, bias, res, out,
                                                                       stream);
}

// Data gradient of the folded up-sampling (tae.py:110-116): 64 taps over the 8 parity views of dy in one launch, no
// epilogue (include/vqb200.h).
extern "C" int vqb_conv3d_dgrad_gemm(const VqbConv3dDgradDesc* d, const void* dy, const void* w_packed, void* dx,
                                     void* stream) {
    VQB_CHECK(d == nullptr || d->flags == 0, "vqb_conv3d_dgrad_gemm: flags 0x%x: the data gradient has no epilogue",
              d->flags);
    return conv3d_impl<VqbConv3dDgradDesc, Conv3dDgradParams, VQB_MAX_TAPS_3D_DGRAD>("vqb_conv3d_dgrad_gemm", d, dy,
                                                                                     w_packed, nullptr, nullptr, dx,
                                                                                     stream);
}
