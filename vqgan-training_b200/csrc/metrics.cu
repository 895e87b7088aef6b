// Reconstruction metrics: per-item PSNR and SSIM of two images [B, C, H, W] or clips [B, C, T, H, W] (DESIGN.md
// section 3.9, definition in section 7 row 25). An item is an image b or a frame (b, t); a clip is scored per frame.
//
// Every value is mapped to u = clamp((v - lo) * inv, 0, 1) on load (data range 1). PSNR = 10 log10(1 / MSE) with MSE the
// mean of (u_x - u_y)^2 over the item's C*H*W values (+inf when MSE = 0). SSIM is Wang et al. 2004 without padding or
// downsampling: the 11x11 Gaussian window (sigma 1.5) at each of the (H-10)(W-10) valid positions of each channel, C1 =
// 0.01^2, C2 = 0.03^2, averaged over channels and positions.
//
// psnr_ssim_tile_kernel: one CTA per kMTile x kMTile block of valid SSIM positions of one (b, c, t) plane, read in
// place from NCHW / NCTHW. The haloed input tile (kMTile + 10)^2 of x and y is mapped into shared memory; the horizontal
// 11-tap pass writes the five moments of a = u_x - 0.5, b = u_y - 0.5 (a, b, a^2, b^2, ab) per input row into shared
// memory, and the vertical pass slides down them, four output rows per thread, and evaluates SSIM. Centring on 0.5
// keeps |a|, |b| <= 0.5, so sigma^2 = E[a^2] - E[a]^2 cancels against 0.25 instead of 1. The same CTA sums (u_x - u_y)^2
// over its share of the plane: input rows [y0, y0 + kMTile) and columns [x0, x0 + kMTile), extended to H (W) for the
// last tile row (column), which the tile's halo covers; the shares partition the plane, so every value counts once.
// The CTA writes its two fp32 partial sums to work[2 * cta]; CTAs are numbered (item, channel, tile) so that an item's
// partials are contiguous.
//
// psnr_ssim_finish_kernel: one CTA per item sums that item's partials in fp64 in a fixed order and writes PSNR and SSIM.
// No atomics anywhere: reruns are bit-identical. The SSIM formula is evaluated with explicitly rounded operations (no
// FMA contraction), so identical inputs give exactly 1.0 at every position.
#include <cmath>
#include <cuda_bf16.h>

#include "common.cuh"

namespace vqb {

constexpr int kMTile = 32;                // valid positions per tile side
constexpr int kMIn = kMTile + 10;         // haloed input tile side
constexpr int kMThreads = 256;            // 8 warps
constexpr int kMRowsPerThread = kMTile / (kMThreads / 32);  // 4 output rows per thread in the vertical pass

struct MetricsWindow {
    float g[11];  // normalised 1-D Gaussian, sigma 1.5, rounded once to fp32
};

template <bool kBf16>
__device__ __forceinline__ float metrics_load(const void* p, int64_t i) {
    if constexpr (kBf16)
        return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
    else
        return static_cast<const float*>(p)[i];
}

template <bool kBf16>
__global__ void __launch_bounds__(kMThreads) psnr_ssim_tile_kernel(const void* __restrict__ x,
                                                                   const void* __restrict__ y, int C, int T, int H,
                                                                   int W, int tiles_x, int tiles_per_plane, float lo,
                                                                   float inv, MetricsWindow win,
                                                                   float* __restrict__ work) {
    __shared__ float sx[kMIn][kMIn];
    __shared__ float sy[kMIn][kMIn];
    __shared__ float hm[5][kMIn][kMTile];
    __shared__ float red[2][kMThreads / 32];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t cta = blockIdx.x;
    const int tile = static_cast<int>(cta % tiles_per_plane);
    const int64_t ic = cta / tiles_per_plane;  // item * C + c
    const int c = static_cast<int>(ic % C);
    const int64_t item = ic / C;               // b * T + t
    const int64_t b = item / T, t = item % T;
    const int64_t plane = ((b * C + c) * T + t) * static_cast<int64_t>(H) * W;
    const int ty = tile / tiles_x, tx = tile % tiles_x;
    const int y0 = ty * kMTile, x0 = tx * kMTile;
    const int Ho = H - 10, Wo = W - 10;

    // haloed tile, mapped on load; values past the plane are 0 and only ever reach invalid positions
    for (int r = warp; r < kMIn; r += kMThreads / 32) {
        const int gy = y0 + r;
        for (int cc = lane; cc < kMIn; cc += 32) {
            const int gx = x0 + cc;
            float ux = 0.f, uy = 0.f;
            if (gy < H && gx < W) {
                const int64_t i = plane + static_cast<int64_t>(gy) * W + gx;
                ux = fminf(fmaxf(__fmul_rn(__fsub_rn(metrics_load<kBf16>(x, i), lo), inv), 0.f), 1.f);
                uy = fminf(fmaxf(__fmul_rn(__fsub_rn(metrics_load<kBf16>(y, i), lo), inv), 0.f), 1.f);
            }
            sx[r][cc] = ux;
            sy[r][cc] = uy;
        }
    }
    __syncthreads();

    // PSNR share: rows [0, own_h) x columns [0, own_w) of the tile
    const int own_h = ty == (Ho - 1) / kMTile ? H - y0 : kMTile;
    const int own_w = tx == tiles_x - 1 ? W - x0 : kMTile;
    float sq = 0.f;
    for (int i = threadIdx.x; i < own_h * own_w; i += kMThreads) {
        const int r = i / own_w, cc = i - r * own_w;
        const float d = __fsub_rn(sx[r][cc], sy[r][cc]);
        sq = __fadd_rn(sq, __fmul_rn(d, d));
    }

    // horizontal pass: moments of every input row at each of the tile's kMTile columns
    for (int r = warp; r < kMIn; r += kMThreads / 32) {
        float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float a = __fsub_rn(sx[r][lane + k], 0.5f), bb = __fsub_rn(sy[r][lane + k], 0.5f);
            const float g = win.g[k];
            m0 = __fmaf_rn(g, a, m0);
            m1 = __fmaf_rn(g, bb, m1);
            m2 = __fmaf_rn(g, __fmul_rn(a, a), m2);
            m3 = __fmaf_rn(g, __fmul_rn(bb, bb), m3);
            m4 = __fmaf_rn(g, __fmul_rn(a, bb), m4);
        }
        hm[0][r][lane] = m0;
        hm[1][r][lane] = m1;
        hm[2][r][lane] = m2;
        hm[3][r][lane] = m3;
        hm[4][r][lane] = m4;
    }
    __syncthreads();

    // vertical pass: output rows i0 .. i0 + 3 of column `lane` slide over input rows i0 .. i0 + 13
    const int i0 = warp * kMRowsPerThread;
    float acc[kMRowsPerThread][5];
#pragma unroll
    for (int q = 0; q < kMRowsPerThread; ++q)
#pragma unroll
        for (int m = 0; m < 5; ++m) acc[q][m] = 0.f;
#pragma unroll
    for (int k = 0; k < 10 + kMRowsPerThread; ++k) {
        float v[5];
#pragma unroll
        for (int m = 0; m < 5; ++m) v[m] = hm[m][i0 + k][lane];
#pragma unroll
        for (int q = 0; q < kMRowsPerThread; ++q) {
            if (k - q >= 0 && k - q <= 10) {
#pragma unroll
                for (int m = 0; m < 5; ++m) acc[q][m] = __fmaf_rn(win.g[k - q], v[m], acc[q][m]);
            }
        }
    }
    constexpr float C1 = 1e-4f, C2 = 9e-4f;  // 0.01^2 and 0.03^2 rounded once
    float ss = 0.f;
#pragma unroll
    for (int q = 0; q < kMRowsPerThread; ++q) {
        if (y0 + i0 + q < Ho && x0 + lane < Wo) {
            const float ma = acc[q][0], mb = acc[q][1];
            const float vx = __fsub_rn(acc[q][2], __fmul_rn(ma, ma));
            const float vy = __fsub_rn(acc[q][3], __fmul_rn(mb, mb));
            const float cxy = __fsub_rn(acc[q][4], __fmul_rn(ma, mb));
            const float mx = __fadd_rn(ma, 0.5f), my = __fadd_rn(mb, 0.5f);
            const float n1 = __fadd_rn(__fmul_rn(2.f, __fmul_rn(mx, my)), C1);
            const float d1 = __fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), C1);
            const float n2 = __fadd_rn(__fmul_rn(2.f, cxy), C2);
            const float d2 = __fadd_rn(__fadd_rn(vx, vy), C2);
            ss = __fadd_rn(ss, __fdiv_rn(__fmul_rn(n1, n2), __fmul_rn(d1, d2)));
        }
    }

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ss = __fadd_rn(ss, __shfl_xor_sync(0xffffffffu, ss, o));
        sq = __fadd_rn(sq, __shfl_xor_sync(0xffffffffu, sq, o));
    }
    if (lane == 0) {
        red[0][warp] = ss;
        red[1][warp] = sq;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int w = 0; w < kMThreads / 32; ++w) {
            s0 = __fadd_rn(s0, red[0][w]);
            s1 = __fadd_rn(s1, red[1][w]);
        }
        work[2 * cta] = s0;
        work[2 * cta + 1] = s1;
    }
}

__global__ void __launch_bounds__(kMThreads) psnr_ssim_finish_kernel(const float* __restrict__ work, int parts,
                                                                     double n_values, double n_positions,
                                                                     float* __restrict__ psnr,
                                                                     float* __restrict__ ssim) {
    __shared__ double red[2][kMThreads];
    const int64_t item = blockIdx.x;
    const float* w = work + 2 * item * parts;
    double s0 = 0.0, s1 = 0.0;
    for (int i = threadIdx.x; i < parts; i += kMThreads) {
        s0 += static_cast<double>(w[2 * i]);
        s1 += static_cast<double>(w[2 * i + 1]);
    }
    red[0][threadIdx.x] = s0;
    red[1][threadIdx.x] = s1;
    __syncthreads();
    for (int h = kMThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            red[0][threadIdx.x] += red[0][threadIdx.x + h];
            red[1][threadIdx.x] += red[1][threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double sq = red[1][0];
        psnr[item] = sq > 0.0 ? static_cast<float>(10.0 * log10(n_values / sq)) : INFINITY;
        ssim[item] = static_cast<float>(red[0][0] / n_positions);
    }
}

}  // namespace vqb

using namespace vqb;

extern "C" {

int vqb_psnr_ssim(const void* x, const void* y, int bf16, int B, int C, int T, int H, int W, float lo, float hi,
                  float* psnr, float* ssim, float* work, int64_t work_elems, void* stream) {
    VQB_CHECK(x && y && psnr && ssim && work, "vqb_psnr_ssim: null pointer");
    VQB_CHECK(bf16 == 0 || bf16 == 1, "vqb_psnr_ssim: bf16 must be 0 or 1, got %d", bf16);
    VQB_CHECK(B > 0 && C > 0 && T > 0, "vqb_psnr_ssim: bad extents B=%d C=%d T=%d", B, C, T);
    VQB_CHECK(H >= 11 && W >= 11, "vqb_psnr_ssim: H=%d and W=%d must be >= 11 (the SSIM window)", H, W);
    VQB_CHECK(std::isfinite(lo) && std::isfinite(hi) && hi > lo,
              "vqb_psnr_ssim: bad value range (%g, %g): need finite lo < hi", lo, hi);
    const int tiles_x = (W - 10 + kMTile - 1) / kMTile, tiles_y = (H - 10 + kMTile - 1) / kMTile;
    const int64_t parts = static_cast<int64_t>(C) * tiles_x * tiles_y;
    const int64_t items = static_cast<int64_t>(B) * T;
    const int64_t ctas = items * parts;
    VQB_CHECK(ctas <= 0x7fffffffLL, "vqb_psnr_ssim: %lld tiles exceed the launch grid", (long long)ctas);
    VQB_CHECK(work_elems >= 2 * ctas, "vqb_psnr_ssim: work holds %lld floats, needs 2 * B * T * C * %d * %d = %lld",
              (long long)work_elems, tiles_y, tiles_x, (long long)(2 * ctas));
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_psnr_ssim: current device is not sm_90");

    MetricsWindow win;
    double g[11], sum = 0.0;
    for (int i = 0; i < 11; ++i) sum += (g[i] = exp(-(i - 5) * (i - 5) / (2.0 * 1.5 * 1.5)));
    for (int i = 0; i < 11; ++i) win.g[i] = static_cast<float>(g[i] / sum);
    const float inv = static_cast<float>(1.0 / (static_cast<double>(hi) - lo));  // 1 / (hi - lo), rounded once
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int tpp = tiles_x * tiles_y;
    if (bf16)
        psnr_ssim_tile_kernel<true><<<static_cast<unsigned>(ctas), kMThreads, 0, st>>>(x, y, C, T, H, W, tiles_x, tpp,
                                                                                       lo, inv, win, work);
    else
        psnr_ssim_tile_kernel<false><<<static_cast<unsigned>(ctas), kMThreads, 0, st>>>(x, y, C, T, H, W, tiles_x, tpp,
                                                                                        lo, inv, win, work);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    psnr_ssim_finish_kernel<<<static_cast<unsigned>(items), kMThreads, 0, st>>>(
        work, static_cast<int>(parts), static_cast<double>(C) * H * W, static_cast<double>(C) * (H - 10) * (W - 10),
        psnr, ssim);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

}  // extern "C"
