// Tiled encode / decode: accumulate one tile's module output into the full [N, C, T, H, W] grid with its separable
// blend weight (DESIGN.md section 3.11, definition in section 7 row 27). tiling.py plans the tiles, computes the per-axis
// weight tables and launches this once per tile in raster order (t, then h, then w).
//
// Per element of the tile at grid coordinates (t, h, w): p = (wt * wh) * ww, rounded in that order. The element is
// this tile's FIRST contribution when every coordinate is >= the axis's prev_end (the end of the previous tile on that
// axis): the tiles covering a point are a product of per-axis index ranges, so the raster-order first contributor is
// the per-axis first on every axis. First: acc = p * v; otherwise acc = fmaf(p, v, acc). It is the LAST contribution when
// every coordinate is < the axis's next_start; then, when a bf16 output is given, out = bf16_rn(acc). So there is no
// memset pass and no atomics, every element is written in launch order (reruns are bit-identical), and each bf16 output
// element is rounded exactly once, by the launch that completes it.
//
// One thread per kVec consecutive elements along W; a grid-stride walk over (row, vector) with row = (n, c, t, h) of
// the tile. 64-bit offsets into the grid. kVec = 4 when the window start, the tile row, the grid row and the pointers
// allow 16-byte (fp32) / 8-byte (bf16) accesses; otherwise the scalar form (latent windows may start anywhere).
#include <cuda_bf16.h>

#include "common.cuh"

namespace vqb {

constexpr int kBThreads = 256;
constexpr int kBMaxBlocks = 8192;

struct BlendAxes {
    int t0, h0, w0;        // window start in the grid
    int pt, ph, pw;        // prev_end per axis
    int nt, nh, nw;        // next_start per axis
};

template <bool kTileBf16>
__device__ __forceinline__ float blend_load(const void* p, int64_t i) {
    if constexpr (kTileBf16)
        return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
    else
        return static_cast<const float*>(p)[i];
}

template <bool kTileBf16>
__device__ __forceinline__ void blend_load4(const void* p, int64_t i, float v[4]) {
    if constexpr (kTileBf16) {
        const uint2 u = *reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(p) + i);
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
        v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y;
    } else {
        const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + i);
        v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w;
    }
}

template <bool kTileBf16, int kVec>
__global__ void __launch_bounds__(kBThreads) tile_blend_kernel(const void* __restrict__ tile, float* __restrict__ acc,
                                                               __nv_bfloat16* __restrict__ out, int T, int H, int W,
                                                               int Lt, int Lh, int Lw, BlendAxes ax,
                                                               const float* __restrict__ wt,
                                                               const float* __restrict__ wh,
                                                               const float* __restrict__ ww, int64_t vpr,
                                                               int64_t work) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(kBThreads) + threadIdx.x; i < work;
         i += static_cast<int64_t>(gridDim.x) * kBThreads) {
        const int64_t row = i / vpr;
        const int w = static_cast<int>(i - row * vpr) * kVec;
        const int h = static_cast<int>(row % Lh);
        const int64_t r2 = row / Lh;
        const int t = static_cast<int>(r2 % Lt);
        const int64_t nc = r2 / Lt;
        const int gt = ax.t0 + t, gh = ax.h0 + h, gw = ax.w0 + w;
        const int64_t g = ((nc * T + gt) * H + gh) * static_cast<int64_t>(W) + gw;
        const int64_t s = row * Lw + w;
        const float pth = __fmul_rn(wt[t], wh[h]);
        const bool first_th = gt >= ax.pt && gh >= ax.ph;
        const bool last_th = gt < ax.nt && gh < ax.nh;
        if constexpr (kVec == 4) {
            float v[4], a[4];
            blend_load4<kTileBf16>(tile, s, v);
            const bool all_first = first_th && gw >= ax.pw;
            if (!all_first) {
                const float4 o = *reinterpret_cast<const float4*>(acc + g);
                a[0] = o.x, a[1] = o.y, a[2] = o.z, a[3] = o.w;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float p = __fmul_rn(pth, ww[w + j]);
                a[j] = (first_th && gw + j >= ax.pw) ? __fmul_rn(p, v[j]) : __fmaf_rn(p, v[j], a[j]);
            }
            *reinterpret_cast<float4*>(acc + g) = make_float4(a[0], a[1], a[2], a[3]);
            if (out != nullptr && last_th) {
                if (gw + 3 < ax.nw) {
                    __nv_bfloat162 b0 = __floats2bfloat162_rn(a[0], a[1]), b1 = __floats2bfloat162_rn(a[2], a[3]);
                    uint2 u;
                    u.x = *reinterpret_cast<uint32_t*>(&b0);
                    u.y = *reinterpret_cast<uint32_t*>(&b1);
                    *reinterpret_cast<uint2*>(out + g) = u;
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (gw + j < ax.nw) out[g + j] = __float2bfloat16_rn(a[j]);
                }
            }
        } else {
            const float v = blend_load<kTileBf16>(tile, s);
            const float p = __fmul_rn(pth, ww[w]);
            const float r = (first_th && gw >= ax.pw) ? __fmul_rn(p, v) : __fmaf_rn(p, v, acc[g]);
            acc[g] = r;
            if (out != nullptr && last_th && gw < ax.nw) out[g] = __float2bfloat16_rn(r);
        }
    }
}

template <bool kTileBf16, int kVec>
static void launch_blend(const void* tile, float* acc, __nv_bfloat16* out, int T, int H, int W, int Lt, int Lh,
                         int Lw, const BlendAxes& ax, const float* wt, const float* wh, const float* ww, int64_t rows,
                         cudaStream_t st) {
    const int64_t vpr = Lw / kVec, work = rows * vpr;
    const int64_t blocks = (work + kBThreads - 1) / kBThreads;
    const unsigned grid = static_cast<unsigned>(blocks < kBMaxBlocks ? blocks : kBMaxBlocks);
    tile_blend_kernel<kTileBf16, kVec><<<grid, kBThreads, 0, st>>>(tile, acc, out, T, H, W, Lt, Lh, Lw, ax, wt, wh, ww,
                                                                   vpr, work);
}

static bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace vqb

using namespace vqb;

extern "C" {

int vqb_tile_blend(const void* tile, int tile_bf16, float* acc, void* out_bf16, int N, int C, int T, int H, int W,
                   int Lt, int Lh, int Lw, int t0, int h0, int w0, const float* wt, const float* wh, const float* ww,
                   int prev_end_t, int prev_end_h, int prev_end_w, int next_start_t, int next_start_h,
                   int next_start_w, void* stream) {
    VQB_CHECK(tile && acc && wt && wh && ww, "vqb_tile_blend: null pointer");
    VQB_CHECK(tile_bf16 == 0 || tile_bf16 == 1, "vqb_tile_blend: tile_bf16 must be 0 or 1, got %d", tile_bf16);
    VQB_CHECK(N > 0 && C > 0 && T > 0 && H > 0 && W > 0, "vqb_tile_blend: bad grid N=%d C=%d T=%d H=%d W=%d", N, C, T,
              H, W);
    VQB_CHECK(Lt > 0 && Lh > 0 && Lw > 0, "vqb_tile_blend: bad tile extents Lt=%d Lh=%d Lw=%d", Lt, Lh, Lw);
    VQB_CHECK(static_cast<double>(N) * C * T * H * W < 4.0e18, "vqb_tile_blend: grid of %g elements is too large",
              static_cast<double>(N) * C * T * H * W);
    const int ext[3] = {T, H, W}, len[3] = {Lt, Lh, Lw}, o[3] = {t0, h0, w0};
    const int pe[3] = {prev_end_t, prev_end_h, prev_end_w}, ns[3] = {next_start_t, next_start_h, next_start_w};
    const char* axis = "THW";
    for (int a = 0; a < 3; ++a) {
        VQB_CHECK(o[a] >= 0 && static_cast<int64_t>(o[a]) + len[a] <= ext[a],
                  "vqb_tile_blend: window [%d, %lld) on axis %c is outside [0, %d)", o[a],
                  static_cast<long long>(o[a]) + len[a], axis[a], ext[a]);
        VQB_CHECK(pe[a] >= o[a] && pe[a] <= o[a] + len[a],
                  "vqb_tile_blend: prev_end %d on axis %c is outside the window [%d, %d]", pe[a], axis[a], o[a],
                  o[a] + len[a]);
        VQB_CHECK(ns[a] >= o[a] && ns[a] <= ext[a],
                  "vqb_tile_blend: next_start %d on axis %c is outside [%d, %d]", ns[a], axis[a], o[a], ext[a]);
    }
    const uintptr_t es = tile_bf16 ? 2 : 4;
    VQB_CHECK(aligned(tile, es) && aligned(acc, 4) && aligned(out_bf16, 2), "vqb_tile_blend: misaligned pointer");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_tile_blend: current device is not sm_90");

    const BlendAxes ax{t0, h0, w0, prev_end_t, prev_end_h, prev_end_w, next_start_t, next_start_h, next_start_w};
    const int64_t rows = static_cast<int64_t>(N) * C * Lt * Lh;
    __nv_bfloat16* out = static_cast<__nv_bfloat16*>(out_bf16);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec = W % 4 == 0 && w0 % 4 == 0 && Lw % 4 == 0 && aligned(tile, 4 * es) && aligned(acc, 16) &&
                     aligned(out_bf16, 8);
    if (tile_bf16) {
        if (vec)
            launch_blend<true, 4>(tile, acc, out, T, H, W, Lt, Lh, Lw, ax, wt, wh, ww, rows, st);
        else
            launch_blend<true, 1>(tile, acc, out, T, H, W, Lt, Lh, Lw, ax, wt, wh, ww, rows, st);
    } else {
        if (vec)
            launch_blend<false, 4>(tile, acc, out, T, H, W, Lt, Lh, Lw, ax, wt, wh, ww, rows, st);
        else
            launch_blend<false, 1>(tile, acc, out, T, H, W, Lt, Lh, Lw, ax, wt, wh, ww, rows, st);
    }
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

}  // extern "C"
