// HBM-bound kernels of the VAE path: layout conversion at the module boundary, weight packing,
// fused GroupNorm(+SiLU / LeakyReLU) forward / backward, LeakyReLU, bias gradients, wgrad split
// reduction. All activations are NHWC bf16 with C % 8 == 0; every thread moves 16-byte vectors and
// owns a FIXED 8-channel slot (its channel vector index never changes while it strides over pixels),
// so per-channel affine terms / reductions stay in registers.
//
// Reference semantics: FP32GroupNorm ae.py:41-53 (32 groups, biased variance, eps inside sqrt,
// fp32 math), swish ae.py:13-14, Upsample ae.py:157-167 (nearest), Conv2d bias gradients.
#ifndef VQB_EXACT_SIGMOID
#define VQB_EXACT_SIGMOID 0
#endif
#include "common.cuh"
#include "ptx.cuh"

namespace vqb {

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 ldg16(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void cvt8(const uint4& u, float (&f)[8]) {
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]);
    u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]);
    u.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(p) = u;
}
// sigmoid(x) = 0.5 + 0.5 tanh(x/2) with the single-instruction MUFU.TANH (abs error of the sigmoid <= ~2.5e-4, an order
// of magnitude below the bf16 rounding of the activations it multiplies): one SFU op instead of ex2 + rcp. The GroupNorm
// kernels are limited by special-function and FP32 issue throughput as much as by HBM bandwidth, so this is time.
__device__ __forceinline__ float sigmoidf_(float x) {
#if VQB_EXACT_SIGMOID
    return 1.f / (1.f + __expf(-x));
#else
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
    return fmaf(0.5f, t, 0.5f);
#endif
}

// activation codes of the GroupNorm entry points (their `int silu` argument)
constexpr int kActNone = 0, kActLeaky = 2;  // 1: swish
// negative slope of the LeakyReLU of the 3-D PatchGAN discriminator (tae_disc.py)
constexpr float kLeakySlope = 0.2f;

// tanh for the swish derivative: MUFU.TANH by default; with -DVQB_EXACT_SIGMOID the exact form through exp
__device__ __forceinline__ float tanh_fast(float x) {
#if VQB_EXACT_SIGMOID
    return 2.f / (1.f + __expf(-2.f * x)) - 1.f;
#else
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(x));
    return t;
#endif
}

// ------------------------------------------------------------------ weight packing
// out[r][slot][k] (bf16), r < R, k < Kpad:  transpose ? w[k][r][tap] : w[r][k][tap]   (w is OIHW fp32 or bf16,
// tap = tapmap[slot] indexes KH*KW), zero for k >= K. From a bf16 master the re-layout is exact.
template <typename Src>
__global__ void pack_weights_kernel(const Src* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cout, int Cin,
                                    int T, int nslots, const int* __restrict__ tapmap, int transpose, int Kpad) {
    const int R = transpose ? Cin : Cout;
    const int K = transpose ? Cout : Cin;
    const int64_t total = static_cast<int64_t>(R) * nslots * Kpad;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(i % Kpad);
        const int slot = static_cast<int>((i / Kpad) % nslots);
        const int r = static_cast<int>(i / (static_cast<int64_t>(Kpad) * nslots));
        float v = 0.f;
        if (k < K) {
            const int tap = tapmap[slot];
            const int co = transpose ? k : r, ci = transpose ? r : k;
            v = to_f32(w[(static_cast<int64_t>(co) * Cin + ci) * T + tap]);
        }
        out[i] = __float2bfloat16(v);
    }
}

// Folded packing: out[r][slot][k] = sum over the taps in tapmask[slot] (bit t = tap t) of w[..][tap]; the fp32 sum is
// rounded to bf16 once (for a bf16 master too). Used by the nearest-2x-upsample + conv3x3 fusion (4 phase convs with
// 2x2 folded taps).
template <typename Src>
__global__ void pack_weights_fold_kernel(const Src* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cout,
                                         int Cin, int T, int nslots, const int* __restrict__ tapmask, int transpose,
                                         int Kpad) {
    const int R = transpose ? Cin : Cout;
    const int K = transpose ? Cout : Cin;
    const int64_t total = static_cast<int64_t>(R) * nslots * Kpad;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(i % Kpad);
        const int slot = static_cast<int>((i / Kpad) % nslots);
        const int r = static_cast<int>(i / (static_cast<int64_t>(Kpad) * nslots));
        float v = 0.f;
        if (k < K) {
            const int mask = tapmask[slot];
            const int co = transpose ? k : r, ci = transpose ? r : k;
            const Src* wp = w + (static_cast<int64_t>(co) * Cin + ci) * T;
            for (int t = 0; t < T; ++t)
                if ((mask >> t) & 1) v += to_f32(wp[t]);
        }
        out[i] = __float2bfloat16(v);
    }
}

// ------------------------------------------------------------------ layout conversion
// y[n,h,w,c] = (x[n,c,h,w] - shift[c]) * inv_scale[c]   (bf16 NHWC, channels >= C zero)
// pad > 0: y is [N][H+2pad][W+2pad][Cpad] (pre-zeroed) and only its interior is written (W needed then)
// x is fp32 or bf16 (a bf16 image enters without an fp32 copy; the affine math is fp32 either way)
template <typename In>
__global__ void nchw_to_nhwc_kernel(const In* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int C, int HW,
                                    int Cpad, const float* __restrict__ shift, const float* __restrict__ inv_scale,
                                    int W, int pad) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    const int H = HW / W;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t n = i / HW, p = i % HW;
        const In* xp = x + n * C * HW + p;
        int64_t opix = i;
        if (pad) {
            const int h = static_cast<int>(p / W), w = static_cast<int>(p % W);
            opix = (n * (H + 2 * pad) + h + pad) * (W + 2 * pad) + w + pad;
        }
        __nv_bfloat16* yp = y + opix * Cpad;
        for (int c0 = 0; c0 < Cpad; c0 += 8) {
            float f[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = c0 + j;
                float v = 0.f;
                if (c < C) {
                    v = to_f32(xp[static_cast<int64_t>(c) * HW]);
                    if (shift) v = (v - shift[c]) * inv_scale[c];
                }
                f[j] = v;
            }
            store8(yp + c0, f);
        }
    }
}

// gx[n,c,h,w] = g[n,h,w,c] * inv_scale[c]   (fp32 or bf16 NCHW out; without inv_scale the bf16 copy is exact)
template <typename Out>
__global__ void nhwc_to_nchw_kernel(const __nv_bfloat16* __restrict__ g, Out* __restrict__ gx, int N, int C, int HW,
                                    int Cpad, const float* __restrict__ inv_scale, int W, int pad) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    const int H = HW / W;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t n = i / HW, p = i % HW;
        int64_t ipix = i;
        if (pad) {
            const int h = static_cast<int>(p / W), w = static_cast<int>(p % W);
            ipix = (n * (H + 2 * pad) + h + pad) * (W + 2 * pad) + w + pad;
        }
        const __nv_bfloat16* gp = g + ipix * Cpad;
        Out* xp = gx + n * C * HW + p;
        for (int c = 0; c < C; ++c) {
            float v = __bfloat162float(gp[c]);
            if (inv_scale) v *= inv_scale[c];
            from_f32(xp[static_cast<int64_t>(c) * HW], v);
        }
    }
}

// ------------------------------------------------------------------ clip <-> per-frame layout
// Clips are NCTHW: channel stride T*HW, frame stride HW. Image i of the per-frame NHWC buffer is frame frames[i] (all
// frames: i % Tsel) of clip i / Tsel. grid (pixel blocks, images); per element the arithmetic of nchw_to_nhwc_kernel.
template <typename In>
__global__ void clip_to_frames_kernel(const In* __restrict__ x, __nv_bfloat16* __restrict__ y, int C, int T, int HW,
                                      int W, int Cpad, int pad, const int* __restrict__ frames, int Tsel,
                                      const float* __restrict__ shift, const float* __restrict__ inv_scale) {
    const int img = blockIdx.y;
    const int t = frames ? frames[img] : img % Tsel;
    const int H = HW / W;
    const In* xb = x + (static_cast<int64_t>(img / Tsel) * C * T + t) * HW;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const int h = p / W, w = p % W;
        const int64_t opix = (static_cast<int64_t>(img) * (H + 2 * pad) + h + pad) * (W + 2 * pad) + w + pad;
        __nv_bfloat16* yp = y + opix * Cpad;
        for (int c0 = 0; c0 < Cpad; c0 += 8) {
            float f[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = c0 + j;
                float v = 0.f;
                if (c < C && static_cast<unsigned>(t) < static_cast<unsigned>(T)) {
                    v = to_f32(xb[static_cast<int64_t>(c) * T * HW + p]);
                    if (shift) v = (v - shift[c]) * inv_scale[c];
                }
                f[j] = v;
            }
            store8(yp + c0, f);
        }
    }
}

// gx[b,c,t,h,w] = g[img,h,w,c] * inv_scale[c] where frames[img] == t within clip b, else 0: grid (pixel blocks, B*T clip
// frames), so every element of the clip gradient is written exactly once by one launch.
__global__ void frames_to_clip_kernel(const __nv_bfloat16* __restrict__ g, float* __restrict__ gx, int C, int T, int HW,
                                      int W, int Cpad, int pad, const int* __restrict__ frames, int Tsel,
                                      const float* __restrict__ inv_scale) {
    __shared__ int s_img;
    const int b = blockIdx.y / T, t = blockIdx.y % T;
    if (threadIdx.x == 0) {
        int img = -1;
        if (frames) {
            for (int j = 0; j < Tsel; ++j)
                if (frames[b * Tsel + j] == t) img = b * Tsel + j;
        } else {
            img = b * Tsel + t;
        }
        s_img = img;
    }
    __syncthreads();
    const int img = s_img;
    const int H = HW / W;
    float* xb = gx + (static_cast<int64_t>(b) * C * T + t) * HW;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        float* xp = xb + p;
        if (img < 0) {
            for (int c = 0; c < C; ++c) xp[static_cast<int64_t>(c) * T * HW] = 0.f;
            continue;
        }
        const int h = p / W, w = p % W;
        const int64_t ipix = (static_cast<int64_t>(img) * (H + 2 * pad) + h + pad) * (W + 2 * pad) + w + pad;
        const __nv_bfloat16* gp = g + ipix * Cpad;
        for (int c = 0; c < C; ++c) {
            float v = __bfloat162float(gp[c]);
            if (inv_scale) v *= inv_scale[c];
            xp[static_cast<int64_t>(c) * T * HW] = v;
        }
    }
}

// ------------------------------------------------------------------ GroupNorm forward
// grid (chunks, N); thread t owns channel vector cv = t % V (V = C/8) and pixel rows t / V + k*R.
// The R row partials of a block are summed in a fixed order (no shared-memory float atomics), so the fp32 chunk sums do
// not depend on thread timing; chunks are combined in double.
__global__ void gn_stats_kernel(const __nv_bfloat16* __restrict__ x, double* __restrict__ sums /* [N][C][2] */, int HW,
                                int C, int pix_per_chunk) {
    extern __shared__ float sm[];  // [R][C][2]
    const int V = C >> 3, R = blockDim.x / V;
    const int cv = threadIdx.x % V, pr = threadIdx.x / V;
    const int n = blockIdx.y;
    float s[8], q[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
    const int p0 = blockIdx.x * pix_per_chunk;
    const int p1 = min(HW, p0 + pix_per_chunk);
    if (pr < R) {
        const __nv_bfloat16* xb = x + (static_cast<int64_t>(n) * HW) * C + cv * 8;
        int p = p0 + pr;
        for (; p + 3 * R < p1; p += 4 * R) {  // 4 independent 16-byte loads in flight per thread
            uint4 u[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) u[k] = ldg16(xb + static_cast<int64_t>(p + k * R) * C);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float f[8];
                cvt8(u[k], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    s[j] += f[j];
                    q[j] += f[j] * f[j];
                }
            }
        }
        for (; p < p1; p += R) {
            float f[8];
            load8(xb + static_cast<int64_t>(p) * C, f);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                s[j] += f[j];
                q[j] += f[j] * f[j];
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sm[(pr * C + cv * 8 + j) * 2] = s[j];
            sm[(pr * C + cv * 8 + j) * 2 + 1] = q[j];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
        float v = 0.f;
        for (int r = 0; r < R; ++r) v += sm[r * 2 * C + i];
        atomicAdd(&sums[static_cast<int64_t>(n) * 2 * C + i], static_cast<double>(v));
    }
}

// mean / rstd per (n, group) from the per-channel double sums.
__global__ void gn_finalize_kernel(const double* __restrict__ sums, float* __restrict__ mr /* [N][G][2] */, int N,
                                   int C, int G, int HW, float eps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * G) return;
    const int n = i / G, g = i % G, cpg = C / G;
    double s = 0, q = 0;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        s += sums[(static_cast<int64_t>(n) * C + c) * 2];
        q += sums[(static_cast<int64_t>(n) * C + c) * 2 + 1];
    }
    const double m = static_cast<double>(cpg) * HW;
    const double mean = s / m;
    double var = q / m - mean * mean;
    if (var < 0) var = 0;
    mr[i * 2] = static_cast<float>(mean);
    mr[i * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
}

// same, from per-channel fp32 sums accumulated by the producing convolution's epilogue (VQB_EPI_STATS)
__global__ void gn_finalize_f32_kernel(const float* __restrict__ sums, float* __restrict__ mr, int N, int C, int G,
                                       int HW, float eps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * G) return;
    const int n = i / G, g = i % G, cpg = C / G;
    double s = 0, q = 0;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        s += static_cast<double>(sums[(static_cast<int64_t>(n) * C + c) * 2]);
        q += static_cast<double>(sums[(static_cast<int64_t>(n) * C + c) * 2 + 1]);
    }
    const double m = static_cast<double>(cpg) * HW;
    const double mean = s / m;
    double var = q / m - mean * mean;
    if (var < 0) var = 0;
    mr[i * 2] = static_cast<float>(mean);
    mr[i * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
}

// LEAKY: y = LeakyReLU(0.2)(u) (activation code 2); otherwise `silu` selects swish (1) or none (0)
template <bool LEAKY>
__global__ void gn_apply_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                const float* __restrict__ mr, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int HW, int C, int G, int pix_per_chunk, int silu) {
    const int V = C >> 3, R = blockDim.x / V;
    const int cv = threadIdx.x % V, pr = threadIdx.x / V;
    if (pr >= R) return;
    const int n = blockIdx.y, cpg = C / G;
    float a[8], b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = cv * 8 + j, g = c / cpg;
        const float mean = mr[(n * G + g) * 2], rstd = mr[(n * G + g) * 2 + 1];
        a[j] = rstd * gamma[c];
        b[j] = beta[c] - mean * a[j];
    }
    const int p0 = blockIdx.x * pix_per_chunk;
    const int p1 = min(HW, p0 + pix_per_chunk);
    const int64_t base = (static_cast<int64_t>(n) * HW) * C + cv * 8;
    int p = p0 + pr;
    for (; p + 3 * R < p1; p += 4 * R) {
        uint4 u4[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) u4[k] = ldg16(x + base + static_cast<int64_t>(p + k * R) * C);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float f[8];
            cvt8(u4[k], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float u = fmaf(a[j], f[j], b[j]);
                f[j] = LEAKY ? (u > 0.f ? u : kLeakySlope * u) : (silu ? u * sigmoidf_(u) : u);
            }
            store8(y + base + static_cast<int64_t>(p + k * R) * C, f);
        }
    }
    for (; p < p1; p += R) {
        float f[8];
        load8(x + base + static_cast<int64_t>(p) * C, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float u = fmaf(a[j], f[j], b[j]);
            f[j] = LEAKY ? (u > 0.f ? u : kLeakySlope * u) : (silu ? u * sigmoidf_(u) : u);
        }
        store8(y + base + static_cast<int64_t>(p) * C, f);
    }
}

// ------------------------------------------------------------------ GroupNorm backward
// per-(n,channel) sums of du and du*xhat, du = dy * act'(u), u = xhat*gamma + beta (LEAKY: act'(u) = u > 0 ? 1 : 0.2,
// with u > 0 tested on the recomputed h = u/2)
template <bool LEAKY>
__global__ void gn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                     const float* __restrict__ mr, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float* __restrict__ cs /* [N][C][2] */, int HW,
                                     int C, int G, int pix_per_chunk, int silu) {
    extern __shared__ float sm[];  // [C][2]
    const int V = C >> 3, R = blockDim.x / V;
    const int cv = threadIdx.x % V, pr = threadIdx.x / V;
    const int n = blockIdx.y, cpg = C / G;
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    if (pr < R) {
        // trimmed form (this kernel sat on the FP32-issue / SFU limit): h = x*a2 + b2 (= u/2), t = tanh(h),
        // 2*silu'(u) = (1 + t)(1 + h - h t); s1 = sum 2du, s2 = sum 2du (x - mean); scaled by 1/2 and rstd/2 at the end
        float mean[8], rstd[8], a2[8], b2[8], s1[8], s2[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = cv * 8 + j, g = c / cpg;
            mean[j] = mr[(n * G + g) * 2];
            rstd[j] = mr[(n * G + g) * 2 + 1];
            const float a = gamma[c] * rstd[j];
            a2[j] = 0.5f * a;
            b2[j] = 0.5f * (beta[c] - mean[j] * a);
            s1[j] = s2[j] = 0.f;
        }
        const int p0 = blockIdx.x * pix_per_chunk;
        const int p1 = min(HW, p0 + pix_per_chunk);
        const int64_t base = (static_cast<int64_t>(n) * HW) * C + cv * 8;
        // 4 pixel rows (8 x 16-byte loads) in flight per thread: with few warps per SM, fewer rows leave the kernel
        // waiting on load latency instead of streaming HBM
        constexpr int U = 4;
        for (int p = p0 + pr; p < p1; p += U * R) {
            uint4 ux[U], ud[U];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const bool in = (p + k * R) < p1;
                ux[k] = in ? ldg16(x + base + static_cast<int64_t>(p + k * R) * C) : make_uint4(0, 0, 0, 0);
                ud[k] = in ? ldg16(dy + base + static_cast<int64_t>(p + k * R) * C) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                if ((p + k * R) >= p1) break;
                float f[8], d[8];
                cvt8(ux[k], f);
                cvt8(ud[k], d);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float du2 = 2.f * d[j];
                    if (LEAKY) {
                        if (!(fmaf(f[j], a2[j], b2[j]) > 0.f)) du2 *= kLeakySlope;
                    } else if (silu) {
                        const float h = fmaf(f[j], a2[j], b2[j]);
                        const float t = tanh_fast(h);
                        const float r = fmaf(-h, t, h + 1.f);
                        du2 = d[j] * fmaf(t, r, r);
                    }
                    s1[j] += du2;
                    s2[j] = fmaf(du2, f[j] - mean[j], s2[j]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            atomicAdd(&sm[(cv * 8 + j) * 2], 0.5f * s1[j]);
            atomicAdd(&sm[(cv * 8 + j) * 2 + 1], 0.5f * rstd[j] * s2[j]);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) atomicAdd(&cs[static_cast<int64_t>(n) * 2 * C + i], sm[i]);
}

// gs[n][g] = (sum_c gamma_c*s1, sum_c gamma_c*s2) / m ; dgamma[c] = sum_n s2 ; dbeta[c] = sum_n s1
__global__ void gn_bwd_finalize_kernel(const float* __restrict__ cs, const float* __restrict__ gamma,
                                       float* __restrict__ gs /* [N][G][2] */, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, int N, int C, int G, int HW) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int cpg = C / G;
    if (i < N * G) {
        const int n = i / G, g = i % G;
        float a = 0.f, b = 0.f;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
            a += gamma[c] * cs[(static_cast<int64_t>(n) * C + c) * 2];
            b += gamma[c] * cs[(static_cast<int64_t>(n) * C + c) * 2 + 1];
        }
        const float m = static_cast<float>(cpg) * HW;
        gs[i * 2] = a / m;
        gs[i * 2 + 1] = b / m;
    }
    if (i < C) {
        float a = 0.f, b = 0.f;
        for (int n = 0; n < N; ++n) {
            a += cs[(static_cast<int64_t>(n) * C + i) * 2];
            b += cs[(static_cast<int64_t>(n) * C + i) * 2 + 1];
        }
        dbeta[i] = a;
        dgamma[i] = b;
    }
}

// dx = rstd * (du*gamma - S1 - xhat*S2) (+ add)
template <bool ADD, int U, bool LEAKY>
__global__ void __launch_bounds__(256, 2)
gn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                    const __nv_bfloat16* __restrict__ add, __nv_bfloat16* __restrict__ dx,
                    const float* __restrict__ mr, const float* __restrict__ gs, const float* __restrict__ gamma,
                    const float* __restrict__ beta, int HW, int C, int G, int pix_per_chunk, int silu,
                    float* __restrict__ colsum /* [C] or null */) {
    extern __shared__ float sm[];  // [C] (only when colsum != null)
    const int V = C >> 3, R = blockDim.x / V;
    const int cv = threadIdx.x % V, pr = threadIdx.x / V;
    if (colsum) {
        for (int i = threadIdx.x; i < C; i += blockDim.x) sm[i] = 0.f;
        __syncthreads();
    }
    if (pr < R) {
        const int n = blockIdx.y, cpg = C / G;
        // trimmed form: dx = 2du * (gamma rstd / 2) - rstd S1 - (x - mean) rstd^2 S2, 2du as in the reduce kernel
        float mean[8], a2[8], b2[8], k0[8], k2[8], cs8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = cv * 8 + j, g = c / cpg;
            mean[j] = mr[(n * G + g) * 2];
            const float rstd = mr[(n * G + g) * 2 + 1];
            const float a = gamma[c] * rstd;
            a2[j] = 0.5f * a;
            b2[j] = 0.5f * (beta[c] - mean[j] * a);
            k0[j] = -rstd * gs[(n * G + g) * 2];
            k2[j] = -rstd * rstd * gs[(n * G + g) * 2 + 1];
            cs8[j] = 0.f;
        }
        const int p0 = blockIdx.x * pix_per_chunk;
        const int p1 = min(HW, p0 + pix_per_chunk);
        const int64_t base = (static_cast<int64_t>(n) * HW) * C + cv * 8;
        // U pixel rows in flight per thread (2 or 3 16-byte loads each): U = 3 without the skip-gradient operand, 2 with it
        for (int pp = p0 + pr; pp < p1; pp += U * R) {
            uint4 ux[U], ud[U], ua[U];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const bool in = (pp + k * R) < p1;
                const int64_t off = base + static_cast<int64_t>(pp + k * R) * C;
                ux[k] = in ? ldg16(x + off) : make_uint4(0, 0, 0, 0);
                ud[k] = in ? ldg16(dy + off) : make_uint4(0, 0, 0, 0);
                if (ADD) ua[k] = in ? ldg16(add + off) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                if ((pp + k * R) >= p1) break;
                float f[8], d[8], r[8];
                cvt8(ux[k], f);
                cvt8(ud[k], d);
                if (ADD) cvt8(ua[k], r);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float du2 = 2.f * d[j];
                    if (LEAKY) {
                        if (!(fmaf(f[j], a2[j], b2[j]) > 0.f)) du2 *= kLeakySlope;
                    } else if (silu) {
                        const float h = fmaf(f[j], a2[j], b2[j]);
                        const float t = tanh_fast(h);
                        const float rr = fmaf(-h, t, h + 1.f);
                        du2 = d[j] * fmaf(t, rr, rr);
                    }
                    float v = fmaf(du2, a2[j], fmaf(f[j] - mean[j], k2[j], k0[j]));
                    if (ADD) v += r[j];
                    f[j] = v;
                    // column sums of the bf16 values actually written (= bias gradient of the conv that produced x)
                    cs8[j] += __bfloat162float(__float2bfloat16(v));
                }
                store8(dx + base + static_cast<int64_t>(pp + k * R) * C, f);
            }
        }
        if (colsum) {
#pragma unroll
            for (int j = 0; j < 8; ++j) atomicAdd(&sm[cv * 8 + j], cs8[j]);
        }
    }
    if (colsum) {
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&colsum[i], sm[i]);
    }
}

// ------------------------------------------------------------------ LeakyReLU(0.2)
// y = x > 0 ? x : 0.2 x over n/8 16-byte vectors of bf16 (one rounding of 0.2 x)
__global__ void leaky_relu_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                      int64_t nvec) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < nvec;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float f[8];
        cvt8(ldg16(x + i * 8), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = f[j] > 0.f ? f[j] : kLeakySlope * f[j];
        store8(y + i * 8, f);
    }
}

// dx = dy * (y > 0 ? 1 : 0.2), gated on the saved output: the slope is positive, so y > 0 exactly where x > 0
__global__ void leaky_relu_bwd_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dy,
                                      __nv_bfloat16* __restrict__ dx, int64_t nvec) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < nvec;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float fy[8], f[8];
        cvt8(ldg16(y + i * 8), fy);
        cvt8(ldg16(dy + i * 8), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = fy[j] > 0.f ? f[j] : kLeakySlope * f[j];
        store8(dx + i * 8, f);
    }
}

// ------------------------------------------------------------------ column sums (bias gradient)
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out /* [C] zeroed */,
                              int64_t P, int C, int pix_per_chunk) {
    extern __shared__ float sm[];  // [C]
    const int V = C >> 3, R = blockDim.x / V;
    const int cv = threadIdx.x % V, pr = threadIdx.x / V;
    for (int i = threadIdx.x; i < C; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    if (pr < R) {
        float s[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = 0.f;
        const int64_t p0 = static_cast<int64_t>(blockIdx.x) * pix_per_chunk;
        const int64_t p1 = min(P, p0 + pix_per_chunk);
        int64_t p = p0 + pr;
        for (; p + 3 * R < p1; p += 4 * R) {
            uint4 u[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) u[k] = ldg16(x + (p + k * R) * C + cv * 8);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float f[8];
                cvt8(u[k], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) s[j] += f[j];
            }
        }
        for (; p < p1; p += R) {
            float f[8];
            load8(x + p * C + cv * 8, f);
#pragma unroll
            for (int j = 0; j < 8; ++j) s[j] += f[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(&sm[cv * 8 + j], s[j]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&out[i], sm[i]);
}

// ------------------------------------------------------------------ wgrad split reduction
// grad[co][ci][tap_src] (+)= sum_s partial[s][co][slot*C64 + ci]   (OIHW fp32; slot -> tap via tapmap;
// several slots may map to the same tap when weights were folded)
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ grad, int ksplit, int Cout,
                                    int CoutPad, int Cin, int T, int nslots, int C64,
                                    const int* __restrict__ tapmap, int accumulate) {
    const int64_t total = static_cast<int64_t>(Cout) * Cin * T;
    const int64_t ld = static_cast<int64_t>(nslots) * C64;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        // ci fastest: coalesced reads of the (ksplit x larger) partial buffer, strided 4-byte writes
        const int ci = static_cast<int>(i % Cin);
        const int tap = static_cast<int>((i / Cin) % T);
        const int co = static_cast<int>(i / (static_cast<int64_t>(T) * Cin));
        float acc = 0.f;
        bool any = false;
        for (int slot = 0; slot < nslots; ++slot) {
            if (tapmap[slot] != tap) continue;
            any = true;
            for (int s = 0; s < ksplit; ++s)
                acc += partial[(static_cast<int64_t>(s) * CoutPad + co) * ld + static_cast<int64_t>(slot) * C64 + ci];
        }
        const int64_t o = (static_cast<int64_t>(co) * Cin + ci) * T + tap;
        if (any || !accumulate) grad[o] = accumulate ? grad[o] + acc : acc;
    }
}

// Folded variant: slot s contributes to every tap in tapmask[s] (transpose of pack_weights_fold).
__global__ void wgrad_reduce_fold_kernel(const float* __restrict__ partial, float* __restrict__ grad, int ksplit,
                                         int Cout, int CoutPad, int Cin, int T, int nslots, int C64,
                                         const int* __restrict__ tapmask) {
    const int64_t total = static_cast<int64_t>(Cout) * Cin * T;
    const int64_t ld = static_cast<int64_t>(nslots) * C64;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int ci = static_cast<int>(i % Cin);
        const int tap = static_cast<int>((i / Cin) % T);
        const int co = static_cast<int>(i / (static_cast<int64_t>(T) * Cin));
        float acc = 0.f;
        for (int slot = 0; slot < nslots; ++slot) {
            if (!((tapmask[slot] >> tap) & 1)) continue;
            for (int s = 0; s < ksplit; ++s)
                acc += partial[(static_cast<int64_t>(s) * CoutPad + co) * ld + static_cast<int64_t>(slot) * C64 + ci];
        }
        grad[(static_cast<int64_t>(co) * Cin + ci) * T + tap] = acc;
    }
}


// ------------------------------------------------------------------ wavelet front-end (utils.py:229-247)
// y[n, ho, wo, c*4 + band] = sum_{i,j < 6} x[n, c, 2ho + i - 2, 2wo + j - 2] * filt[band][i][j]   (zero outside):
// the reference's F.pad(2) + grouped 6x6 stride-2 conv, fused with the NCHW fp32 -> NHWC bf16 layout conversion the
// encoder's first conv needs. One thread per output pixel; the 6x6 windows of neighbouring pixels overlap 9x, which the
// L1/L2 absorbs (the whole input batch is a few tens of MB). x is fp32 or bf16; the filter sums are fp32 either way.
template <typename In>
__global__ void wavelet_fwd_kernel(const In* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                   const float* __restrict__ filt, int N, int C, int H, int W, int Cpad) {
    __shared__ float f[4 * 36];
    for (int i = threadIdx.x; i < 144; i += blockDim.x) f[i] = filt[i];
    __syncthreads();
    const int Ho = H / 2, Wo = W / 2;
    const int64_t total = static_cast<int64_t>(N) * Ho * Wo;
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < total;
         p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int wo = static_cast<int>(p % Wo), ho = static_cast<int>((p / Wo) % Ho);
        const int64_t n = p / (static_cast<int64_t>(Wo) * Ho);
        __nv_bfloat16* yp = y + p * Cpad;
        for (int c = 0; c < C; ++c) {
            const In* xp = x + (n * C + c) * static_cast<int64_t>(H) * W;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                const int h = 2 * ho + i - 2;
                if (h < 0 || h >= H) continue;
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    const int w = 2 * wo + j - 2;
                    if (w < 0 || w >= W) continue;
                    const float v = to_f32(__ldg(xp + static_cast<int64_t>(h) * W + w));
#pragma unroll
                    for (int b = 0; b < 4; ++b) acc[b] = fmaf(v, f[b * 36 + i * 6 + j], acc[b]);
                }
            }
#pragma unroll
            for (int b = 0; b < 4; ++b) yp[c * 4 + b] = __float2bfloat16(acc[b]);
        }
        for (int c = 4 * C; c < Cpad; ++c) yp[c] = __float2bfloat16(0.f);
    }
}

static inline int gs_blocks(int64_t total, int threads) {
    int64_t b = (total + threads - 1) / threads;
    const int64_t cap = static_cast<int64_t>(num_sms() > 0 ? num_sms() : 132) * 16;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return static_cast<int>(b);
}

// thread-block shape for the "fixed channel vector" kernels
static inline int cv_threads(int C) {
    const int V = C / 8;
    int t = (256 / V) * V;
    if (t < V) t = V;
    return t;
}
// Grid for the fixed-channel-vector kernels: (chunks, N) blocks of cv_threads(C) threads. The block count is made a
// whole number of waves for the kernel's actual occupancy (these kernels are HBM bound; a 60 %-full second wave was
// costing ~20 %), with at least 4 row-iterations of work per thread.
template <typename Kernel>
static inline void cv_grid(int HW, int C, int N, Kernel kernel, size_t smem, int& chunks, int& pix_per_chunk) {
    const int V = C / 8;
    const int T = cv_threads(C);
    const int R = T / V > 0 ? T / V : 1;
    int bpsm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bpsm, kernel, T, smem) != cudaSuccess || bpsm < 1) bpsm = 4;
    const int concurrent = (num_sms() > 0 ? num_sms() : 132) * bpsm;
    const int min_ppc = R * 4;
    int best_chunks = 1;
    for (int waves = 1; waves <= 8; ++waves) {
        int c = (concurrent * waves) / N;  // chunks per image so that N*c <= waves*concurrent
        if (c < 1) c = 1;
        const int ppc = (HW + c - 1) / c;
        best_chunks = c;
        if (ppc <= 2048 || ppc <= min_ppc) break;  // small enough pieces: stop adding waves
    }
    int ppc = (HW + best_chunks - 1) / best_chunks;
    if (ppc < min_ppc) ppc = min_ppc;
    ppc = ((ppc + R - 1) / R) * R;
    pix_per_chunk = ppc;
    chunks = (HW + ppc - 1) / ppc;
}

// tae.DiagonalGaussian (tae.py:259-264): out = mean + exp(0.5 * max(logvar, -3)) * eps over NCTHW z = [N][2Z][S],
// computed in fp32 and rounded once to the module's dtype.
template <typename T>
__global__ void gauss_reparam_kernel(const T* __restrict__ z, const T* __restrict__ eps, T* __restrict__ out, int Z,
                                     int64_t S, int64_t total) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t s = i % S, nc = i / S;  // nc = n * Z + c
        const int64_t n = nc / Z, c = nc % Z;
        const int64_t zm = (n * 2 * Z + c) * S + s;
        const float mean = to_f32(z[zm]);
        const float logvar = fmaxf(to_f32(z[zm + static_cast<int64_t>(Z) * S]), -3.f);
        from_f32(out[i], fmaf(expf(0.5f * logvar), to_f32(eps[i]), mean));
    }
}

// Backward of gauss_reparam_kernel (fp32 training): dz[n][c] = g (mean half), dz[n][Z + c] = g * eps * 0.5 *
// exp(0.5 * logvar) where logvar >= -3, else 0 (torch's clamp backward passes the gradient at exactly -3).
__global__ void gauss_reparam_bwd_kernel(const float* __restrict__ g, const float* __restrict__ z,
                                         const float* __restrict__ eps, float* __restrict__ dz, int Z, int64_t S,
                                         int64_t total) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t s = i % S, nc = i / S;
        const int64_t n = nc / Z, c = nc % Z;
        const int64_t zm = (n * 2 * Z + c) * S + s, zl = zm + static_cast<int64_t>(Z) * S;
        const float gv = g[i];
        const float lv = z[zl];
        dz[zm] = gv;
        dz[zl] = lv >= -3.f ? gv * eps[i] * expf(0.5f * lv) * 0.5f : 0.f;
    }
}

// Clip boundary (per-frame LPIPS / PatchGAN on NCTHW clips): frames of a clip <-> per-frame NHWC images. `images` is
// the grid's y extent (B*Tsel forward, B*T backward). Every argument is checked before the device.
int check_clip_args(const char* fn, const void* in, const void* out, int B, int C, int T, int H, int W, int Cpad,
                    int pad, const int* frames, int Tsel, const float* shift, const float* inv_scale, int64_t images) {
    VQB_CHECK(in, "%s: null input pointer", fn);
    VQB_CHECK(out, "%s: null output pointer", fn);
    VQB_CHECK(B > 0 && C > 0 && T > 0 && H > 0 && W > 0, "%s: bad clip size (B=%d C=%d T=%d H=%d W=%d)", fn, B, C, T, H,
              W);
    VQB_CHECK(Cpad % 8 == 0 && Cpad >= C, "%s: bad Cpad=%d for C=%d", fn, Cpad, C);
    VQB_CHECK(pad >= 0, "%s: bad pad=%d", fn, pad);
    VQB_CHECK(Tsel > 0 && Tsel <= T, "%s: bad Tsel=%d for T=%d", fn, Tsel, T);
    VQB_CHECK(frames != nullptr || Tsel == T, "%s: Tsel=%d without a frame list must equal T=%d", fn, Tsel, T);
    VQB_CHECK((shift == nullptr) == (inv_scale == nullptr), "%s: shift and inv_scale must both be given or null", fn);
    VQB_CHECK(images <= 65535, "%s: %lld frames in one launch exceed 65535", fn, static_cast<long long>(images));
    VQB_CHECK(static_cast<int64_t>(H) * W <= INT32_MAX / 2, "%s: frame of %dx%d too large", fn, H, W);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "%s: current device is not sm_90", fn);
    return VQB_OK;
}

inline dim3 clip_grid(int HW, int images) {
    const int bx = (HW + 255) / 256;
    return dim3(static_cast<unsigned>(bx < 64 ? bx : 64), static_cast<unsigned>(images));
}

template <typename In>
int clip_to_frames(const char* fn, const In* x, void* y, int B, int C, int T, int H, int W, int Cpad, int pad,
                   const int* frames, int Tsel, const float* shift, const float* inv_scale, void* stream) {
    const int rc = check_clip_args(fn, x, y, B, C, T, H, W, Cpad, pad, frames, Tsel, shift, inv_scale,
                                   static_cast<int64_t>(B) * Tsel);
    if (rc != VQB_OK) return rc;
    clip_to_frames_kernel<In><<<clip_grid(H * W, B * Tsel), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<__nv_bfloat16*>(y), C, T, H * W, W, Cpad, pad, frames, Tsel, shift, inv_scale);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int frames_to_clip(const char* fn, const void* g, float* gx, int B, int C, int T, int H, int W, int Cpad, int pad,
                   const int* frames, int Tsel, const float* inv_scale, void* stream) {
    const int rc = check_clip_args(fn, g, gx, B, C, T, H, W, Cpad, pad, frames, Tsel, inv_scale, inv_scale,
                                   static_cast<int64_t>(B) * T);
    if (rc != VQB_OK) return rc;
    frames_to_clip_kernel<<<clip_grid(H * W, B * T), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(g), gx, C, T, H * W, W, Cpad, pad, frames, Tsel, inv_scale);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

}  // namespace vqb

using namespace vqb;

extern "C" {

int vqb_pack_weights(const float* w, void* out, int Cout, int Cin, int T, int nslots, const int* tapmap_dev,
                     int transpose, int Kpad, void* stream) {
    VQB_CHECK(w && out && tapmap_dev, "vqb_pack_weights: null pointer");
    VQB_CHECK(Kpad % 8 == 0 && Kpad >= (transpose ? Cout : Cin), "vqb_pack_weights: bad Kpad=%d", Kpad);
    const int R = transpose ? Cin : Cout;
    const int64_t total = static_cast<int64_t>(R) * nslots * Kpad;
    pack_weights_kernel<float><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        w, static_cast<__nv_bfloat16*>(out), Cout, Cin, T, nslots, tapmap_dev, transpose, Kpad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_pack_weights_fold(const float* w, void* out, int Cout, int Cin, int T, int nslots, const int* tapmask_dev,
                          int transpose, int Kpad, void* stream) {
    VQB_CHECK(w && out && tapmask_dev, "vqb_pack_weights_fold: null pointer");
    VQB_CHECK(Kpad % 8 == 0 && Kpad >= (transpose ? Cout : Cin) && T <= 31, "vqb_pack_weights_fold: bad Kpad/T");
    const int R = transpose ? Cin : Cout;
    const int64_t total = static_cast<int64_t>(R) * nslots * Kpad;
    pack_weights_fold_kernel<float><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        w, static_cast<__nv_bfloat16*>(out), Cout, Cin, T, nslots, tapmask_dev, transpose, Kpad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// bf16 OIHW masters (inference-only modules): same layouts as vqb_pack_weights / vqb_pack_weights_fold
int vqb_pack_weights_bf16(const void* w, void* out, int Cout, int Cin, int T, int nslots, const int* tapmap_dev,
                          int transpose, int Kpad, void* stream) {
    VQB_CHECK(w && out && tapmap_dev, "vqb_pack_weights_bf16: null pointer");
    VQB_CHECK(Cout > 0 && Cin > 0 && T > 0 && nslots > 0 && Kpad % 8 == 0 && Kpad >= (transpose ? Cout : Cin),
              "vqb_pack_weights_bf16: bad shape (Cout=%d Cin=%d T=%d nslots=%d Kpad=%d)", Cout, Cin, T, nslots, Kpad);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_pack_weights_bf16: current device is not sm_90");
    const int R = transpose ? Cin : Cout;
    const int64_t total = static_cast<int64_t>(R) * nslots * Kpad;
    pack_weights_kernel<__nv_bfloat16><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(w), static_cast<__nv_bfloat16*>(out), Cout, Cin, T, nslots, tapmap_dev,
        transpose, Kpad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_pack_weights_fold_bf16(const void* w, void* out, int Cout, int Cin, int T, int nslots,
                               const int* tapmask_dev, int transpose, int Kpad, void* stream) {
    VQB_CHECK(w && out && tapmask_dev, "vqb_pack_weights_fold_bf16: null pointer");
    VQB_CHECK(Cout > 0 && Cin > 0 && T > 0 && T <= 31 && nslots > 0 && Kpad % 8 == 0 &&
                  Kpad >= (transpose ? Cout : Cin),
              "vqb_pack_weights_fold_bf16: bad shape (Cout=%d Cin=%d T=%d nslots=%d Kpad=%d)", Cout, Cin, T, nslots,
              Kpad);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_pack_weights_fold_bf16: current device is not sm_90");
    const int R = transpose ? Cin : Cout;
    const int64_t total = static_cast<int64_t>(R) * nslots * Kpad;
    pack_weights_fold_kernel<__nv_bfloat16><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(w), static_cast<__nv_bfloat16*>(out), Cout, Cin, T, nslots, tapmask_dev,
        transpose, Kpad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_wgrad_reduce_fold(const float* partial, float* grad, int ksplit, int Cout, int CoutPad, int Cin, int T,
                          int nslots, int C64, const int* tapmask_dev, void* stream) {
    VQB_CHECK(partial && grad && tapmask_dev && T <= 31, "vqb_wgrad_reduce_fold: bad arguments");
    const int64_t total = static_cast<int64_t>(Cout) * Cin * T;
    wgrad_reduce_fold_kernel<<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        partial, grad, ksplit, Cout, CoutPad, Cin, T, nslots, C64, tapmask_dev);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_nchw_to_nhwc(const float* x, void* y, int N, int C, int H, int W, int Cpad, const float* shift,
                     const float* inv_scale, void* stream) {
    VQB_CHECK(x && y && Cpad % 8 == 0 && Cpad >= C, "vqb_nchw_to_nhwc: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * H * W;
    nchw_to_nhwc_kernel<float><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<__nv_bfloat16*>(y), N, C, H * W, Cpad, shift, inv_scale, W, 0);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// bf16 NCHW input (bf16 modules / bf16 images): plain (pad = 0) or into the interior of a PRE-ZEROED framed buffer
int vqb_nchw_to_nhwc_pad_bf16(const void* x, void* y, int N, int C, int H, int W, int Cpad, int pad,
                              const float* shift, const float* inv_scale, void* stream) {
    VQB_CHECK(x && y && N > 0 && C > 0 && H > 0 && W > 0 && Cpad % 8 == 0 && Cpad >= C && pad >= 0 &&
                  (shift == nullptr) == (inv_scale == nullptr),
              "vqb_nchw_to_nhwc_pad_bf16: bad arguments");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_nchw_to_nhwc_pad_bf16: current device is not sm_90");
    const int64_t total = static_cast<int64_t>(N) * H * W;
    nchw_to_nhwc_kernel<__nv_bfloat16><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), N, C, H * W, Cpad, shift, inv_scale, W,
        pad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_nchw_to_nhwc_bf16(const void* x, void* y, int N, int C, int H, int W, int Cpad, const float* shift,
                          const float* inv_scale, void* stream) {
    return vqb_nchw_to_nhwc_pad_bf16(x, y, N, C, H, W, Cpad, 0, shift, inv_scale, stream);
}

// bf16 NHWC -> bf16 NCHW (the module-boundary output of a bf16 module; an exact copy)
int vqb_nhwc_to_nchw_bf16(const void* y, void* x, int N, int C, int H, int W, int Cpad, void* stream) {
    VQB_CHECK(y && x && N > 0 && C > 0 && H > 0 && W > 0 && Cpad % 8 == 0 && Cpad >= C,
              "vqb_nhwc_to_nchw_bf16: bad arguments");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_nhwc_to_nchw_bf16: current device is not sm_90");
    const int64_t total = static_cast<int64_t>(N) * H * W;
    nhwc_to_nchw_kernel<__nv_bfloat16><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(y), static_cast<__nv_bfloat16*>(x), N, C, H * W, Cpad, nullptr, W, 0);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// Same, into the interior of a PRE-ZEROED [N][H+2pad][W+2pad][Cpad] buffer (zero frame for the "fat pixel" first-layer conv)
int vqb_nchw_to_nhwc_pad(const float* x, void* y, int N, int C, int H, int W, int Cpad, int pad, const float* shift,
                         const float* inv_scale, void* stream) {
    VQB_CHECK(x && y && Cpad % 8 == 0 && Cpad >= C && pad >= 0, "vqb_nchw_to_nhwc_pad: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * H * W;
    nchw_to_nhwc_kernel<float><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<__nv_bfloat16*>(y), N, C, H * W, Cpad, shift, inv_scale, W, pad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// inverse: reads the interior of a padded NHWC buffer
int vqb_nhwc_to_nchw_pad(const void* g, float* gx, int N, int C, int H, int W, int Cpad, int pad,
                         const float* inv_scale, void* stream) {
    VQB_CHECK(g && gx && Cpad % 8 == 0 && Cpad >= C && pad >= 0, "vqb_nhwc_to_nchw_pad: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * H * W;
    nhwc_to_nchw_kernel<float><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(g), gx, N, C, H * W, Cpad, inv_scale, W, pad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_nhwc_to_nchw(const void* g, float* gx, int N, int C, int H, int W, int Cpad, const float* inv_scale,
                     void* stream) {
    VQB_CHECK(g && gx && Cpad % 8 == 0 && Cpad >= C, "vqb_nhwc_to_nchw: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * H * W;
    nhwc_to_nchw_kernel<float><<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(g), gx, N, C, H * W, Cpad, inv_scale, W, 0);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_ncthw_frames_to_nhwc_pad(const float* x, void* y, int B, int C, int T, int H, int W, int Cpad, int pad,
                                 const int* frames, int Tsel, const float* shift, const float* inv_scale,
                                 void* stream) {
    return clip_to_frames("vqb_ncthw_frames_to_nhwc_pad", x, y, B, C, T, H, W, Cpad, pad, frames, Tsel, shift,
                          inv_scale, stream);
}

int vqb_ncthw_frames_to_nhwc_pad_bf16(const void* x, void* y, int B, int C, int T, int H, int W, int Cpad, int pad,
                                      const int* frames, int Tsel, const float* shift, const float* inv_scale,
                                      void* stream) {
    return clip_to_frames("vqb_ncthw_frames_to_nhwc_pad_bf16", static_cast<const __nv_bfloat16*>(x), y, B, C, T, H, W,
                          Cpad, pad, frames, Tsel, shift, inv_scale, stream);
}

int vqb_ncthw_frames_to_nhwc(const float* x, void* y, int B, int C, int T, int H, int W, int Cpad, const int* frames,
                             int Tsel, const float* shift, const float* inv_scale, void* stream) {
    return clip_to_frames("vqb_ncthw_frames_to_nhwc", x, y, B, C, T, H, W, Cpad, 0, frames, Tsel, shift, inv_scale,
                          stream);
}

int vqb_ncthw_frames_to_nhwc_bf16(const void* x, void* y, int B, int C, int T, int H, int W, int Cpad,
                                  const int* frames, int Tsel, const float* shift, const float* inv_scale,
                                  void* stream) {
    return clip_to_frames("vqb_ncthw_frames_to_nhwc_bf16", static_cast<const __nv_bfloat16*>(x), y, B, C, T, H, W,
                          Cpad, 0, frames, Tsel, shift, inv_scale, stream);
}

int vqb_nhwc_pad_frames_to_ncthw(const void* g, float* gx, int B, int C, int T, int H, int W, int Cpad, int pad,
                                 const int* frames, int Tsel, const float* inv_scale, void* stream) {
    return frames_to_clip("vqb_nhwc_pad_frames_to_ncthw", g, gx, B, C, T, H, W, Cpad, pad, frames, Tsel, inv_scale,
                          stream);
}

int vqb_nhwc_frames_to_ncthw(const void* g, float* gx, int B, int C, int T, int H, int W, int Cpad, const int* frames,
                             int Tsel, const float* inv_scale, void* stream) {
    return frames_to_clip("vqb_nhwc_frames_to_ncthw", g, gx, B, C, T, H, W, Cpad, 0, frames, Tsel, inv_scale, stream);
}

// the apply pass of every GroupNorm forward entry point; act: a validated activation code
static void launch_gn_apply(const void* x, void* y, const float* mr, const float* gamma, const float* beta, int N,
                            int HW, int C, int G, int act, cudaStream_t st) {
    int chunks, ppc;
    const int T = cv_threads(C);
    const auto* xb = static_cast<const __nv_bfloat16*>(x);
    auto* yb = static_cast<__nv_bfloat16*>(y);
    if (act == kActLeaky) {
        cv_grid(HW, C, N, gn_apply_kernel<true>, 0, chunks, ppc);
        gn_apply_kernel<true><<<dim3(chunks, N), T, 0, st>>>(xb, yb, mr, gamma, beta, HW, C, G, ppc, act);
    } else {
        cv_grid(HW, C, N, gn_apply_kernel<false>, 0, chunks, ppc);
        gn_apply_kernel<false><<<dim3(chunks, N), T, 0, st>>>(xb, yb, mr, gamma, beta, HW, C, G, ppc, act);
    }
}

// GroupNorm(+SiLU) forward. ws: >= N*C*2 doubles (zeroed here); mr: [N][G][2] floats (mean, rstd) kept for backward.
int vqb_gn_silu_fwd(const void* x, void* y, const float* gamma, const float* beta, float* mr, double* ws, int N,
                    int HW, int C, int G, float eps, int silu, void* stream) {
    VQB_CHECK(x && y && gamma && beta && mr && ws, "vqb_gn_silu_fwd: null pointer");
    VQB_CHECK(C % 8 == 0 && C % G == 0 && C <= 2048, "vqb_gn_silu_fwd: C=%d G=%d unsupported", C, G);
    VQB_CHECK(silu >= kActNone && silu <= kActLeaky,
              "vqb_gn_silu_fwd: activation code %d unsupported (0 none, 1 swish, 2 LeakyReLU(0.2))", silu);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_gn_silu_fwd: current device is not sm_90");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    VQB_CUDA(cudaMemsetAsync(ws, 0, sizeof(double) * 2 * N * C, st));
    int chunks, ppc;
    const int T = cv_threads(C);
    const size_t stats_smem = static_cast<size_t>(T / (C / 8)) * 2 * C * sizeof(float);  // [R][C][2]
    cv_grid(HW, C, N, gn_stats_kernel, stats_smem, chunks, ppc);
    gn_stats_kernel<<<dim3(chunks, N), T, stats_smem, st>>>(static_cast<const __nv_bfloat16*>(x), ws, HW, C,
                                                                        ppc);
    gn_finalize_kernel<<<(N * G + 127) / 128, 128, 0, st>>>(ws, mr, N, C, G, HW, eps);
    launch_gn_apply(x, y, mr, gamma, beta, N, HW, C, G, silu, st);
    VQB_CUDA(cudaGetLastError());
    count_launch(3);
    return VQB_OK;
}

// GroupNorm(+SiLU) apply pass alone, with the mean/rstd mr [N][G][2] of an earlier vqb_gn_silu_fwd: the same kernel and
// grid as that call's apply pass, so y is bit-identical to its y (the ResnetBlock recompute of tae.py).
int vqb_gn_silu_apply(const void* x, void* y, const float* gamma, const float* beta, const float* mr, int N, int HW,
                      int C, int G, int silu, void* stream) {
    VQB_CHECK(x && y && gamma && beta && mr, "vqb_gn_silu_apply: null pointer");
    VQB_CHECK(N > 0 && HW > 0 && G > 0 && C % 8 == 0 && C % G == 0 && C <= 2048 && (silu == 0 || silu == 1),
              "vqb_gn_silu_apply: N=%d HW=%d C=%d G=%d silu=%d unsupported", N, HW, C, G, silu);
    VQB_CHECK(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15u) == 0 &&
                  ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta) |
                    reinterpret_cast<uintptr_t>(mr)) & 3u) == 0,
              "vqb_gn_silu_apply: x and y must be 16-byte aligned, gamma, beta and mr 4-byte aligned");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_gn_silu_apply: current device is not sm_90");
    launch_gn_apply(x, y, mr, gamma, beta, N, HW, C, G, silu, static_cast<cudaStream_t>(stream));
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// GroupNorm(+SiLU) forward when the per-(n, channel) sums [N][C][2] (sum, sum of squares; fp32) were already produced by
// the convolution that wrote x (vqb_conv_gemm with VQB_EPI_STATS): finalise + one apply pass, no statistics pass.
int vqb_gn_silu_fwd_pre(const void* x, void* y, const float* gamma, const float* beta, float* mr, const float* chsums,
                        int N, int HW, int C, int G, float eps, int silu, void* stream) {
    VQB_CHECK(x && y && gamma && beta && mr && chsums, "vqb_gn_silu_fwd_pre: null pointer");
    VQB_CHECK(C % 8 == 0 && C % G == 0 && C <= 2048, "vqb_gn_silu_fwd_pre: C=%d G=%d unsupported", C, G);
    VQB_CHECK(silu >= kActNone && silu <= kActLeaky,
              "vqb_gn_silu_fwd_pre: activation code %d unsupported (0 none, 1 swish, 2 LeakyReLU(0.2))", silu);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_gn_silu_fwd_pre: current device is not sm_90");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    gn_finalize_f32_kernel<<<(N * G + 127) / 128, 128, 0, st>>>(chsums, mr, N, C, G, HW, eps);
    launch_gn_apply(x, y, mr, gamma, beta, N, HW, C, G, silu, st);
    VQB_CUDA(cudaGetLastError());
    count_launch(2);
    return VQB_OK;
}

// GroupNorm(+SiLU) backward. ws: >= N*C*2 + N*G*2 floats. dx may alias dy. add (optional) is summed into dx.
// dx_colsum (optional, [C] fp32, overwritten): per-channel sums of dx over all N*HW pixels, i.e. the bias gradient of the
// convolution whose output this GroupNorm normalised, produced in the same pass instead of by vqb_colsum.
int vqb_gn_silu_bwd(const void* x, const void* dy, const void* add, void* dx, const float* gamma, const float* beta,
                    const float* mr, float* dgamma, float* dbeta, float* ws, int N, int HW, int C, int G, int silu,
                    float* dx_colsum, void* stream) {
    VQB_CHECK(x && dy && dx && gamma && beta && mr && dgamma && dbeta && ws, "vqb_gn_silu_bwd: null pointer");
    VQB_CHECK(C % 8 == 0 && C % G == 0 && C <= 2048, "vqb_gn_silu_bwd: C=%d G=%d unsupported", C, G);
    VQB_CHECK(silu >= kActNone && silu <= kActLeaky,
              "vqb_gn_silu_bwd: activation code %d unsupported (0 none, 1 swish, 2 LeakyReLU(0.2))", silu);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_gn_silu_bwd: current device is not sm_90");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int chunks, ppc;
    const int T = cv_threads(C);
    float* cs = ws;                                      // [N][C][2]
    float* gsum = ws + static_cast<int64_t>(N) * C * 2;  // [N][G][2]
    VQB_CUDA(cudaMemsetAsync(cs, 0, sizeof(float) * 2 * N * C, st));
    const bool leaky = silu == kActLeaky;
    const auto* xb = static_cast<const __nv_bfloat16*>(x);
    const auto* dyb = static_cast<const __nv_bfloat16*>(dy);
    if (leaky) {
        cv_grid(HW, C, N, gn_bwd_reduce_kernel<true>, 2 * C * sizeof(float), chunks, ppc);
        gn_bwd_reduce_kernel<true><<<dim3(chunks, N), T, 2 * C * sizeof(float), st>>>(xb, dyb, mr, gamma, beta, cs,
                                                                                       HW, C, G, ppc, silu);
    } else {
        cv_grid(HW, C, N, gn_bwd_reduce_kernel<false>, 2 * C * sizeof(float), chunks, ppc);
        gn_bwd_reduce_kernel<false><<<dim3(chunks, N), T, 2 * C * sizeof(float), st>>>(xb, dyb, mr, gamma, beta, cs,
                                                                                        HW, C, G, ppc, silu);
    }
    count_launch();
    const int fin = (N * G > C ? N * G : C);
    gn_bwd_finalize_kernel<<<(fin + 127) / 128, 128, 0, st>>>(cs, gamma, gsum, dgamma, dbeta, N, C, G, HW);
    const size_t cs_smem = dx_colsum ? C * sizeof(float) : 0;
    if (dx_colsum) VQB_CUDA(cudaMemsetAsync(dx_colsum, 0, sizeof(float) * C, st));
    const auto* ab = static_cast<const __nv_bfloat16*>(add);
    auto* dxb = static_cast<__nv_bfloat16*>(dx);
    if (add && leaky) {
        cv_grid(HW, C, N, gn_bwd_apply_kernel<true, 2, true>, cs_smem, chunks, ppc);
        gn_bwd_apply_kernel<true, 2, true><<<dim3(chunks, N), T, cs_smem, st>>>(
            xb, dyb, ab, dxb, mr, gsum, gamma, beta, HW, C, G, ppc, silu, dx_colsum);
    } else if (add) {
        cv_grid(HW, C, N, gn_bwd_apply_kernel<true, 2, false>, cs_smem, chunks, ppc);
        gn_bwd_apply_kernel<true, 2, false><<<dim3(chunks, N), T, cs_smem, st>>>(
            xb, dyb, ab, dxb, mr, gsum, gamma, beta, HW, C, G, ppc, silu, dx_colsum);
    } else if (leaky) {
        cv_grid(HW, C, N, gn_bwd_apply_kernel<false, 3, true>, cs_smem, chunks, ppc);
        gn_bwd_apply_kernel<false, 3, true><<<dim3(chunks, N), T, cs_smem, st>>>(
            xb, dyb, nullptr, dxb, mr, gsum, gamma, beta, HW, C, G, ppc, silu, dx_colsum);
    } else {
        cv_grid(HW, C, N, gn_bwd_apply_kernel<false, 3, false>, cs_smem, chunks, ppc);
        gn_bwd_apply_kernel<false, 3, false><<<dim3(chunks, N), T, cs_smem, st>>>(
            xb, dyb, nullptr, dxb, mr, gsum, gamma, beta, HW, C, G, ppc, silu, dx_colsum);
    }
    VQB_CUDA(cudaGetLastError());
    count_launch(2);
    return VQB_OK;
}

static int leaky_check(const char* fn, const void* a, const void* b, const void* c, int64_t n) {
    VQB_CHECK(a && b && c, "%s: null pointer", fn);
    VQB_CHECK(n > 0 && n % 8 == 0, "%s: n=%lld must be a positive multiple of 8", fn, static_cast<long long>(n));
    VQB_CHECK(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) &
               15u) == 0,
              "%s: pointers must be 16-byte aligned", fn);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "%s: current device is not sm_90", fn);
    return VQB_OK;
}

// LeakyReLU(0.2) forward over n bf16 elements (see include/vqb200.h)
int vqb_leaky_relu_fwd(const void* x, void* y, int64_t n, void* stream) {
    const int rc = leaky_check("vqb_leaky_relu_fwd", x, y, y, n);
    if (rc != VQB_OK) return rc;
    leaky_relu_fwd_kernel<<<gs_blocks(n / 8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n / 8);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_leaky_relu_bwd(const void* y, const void* dy, void* dx, int64_t n, void* stream) {
    const int rc = leaky_check("vqb_leaky_relu_bwd", y, dy, dx, n);
    if (rc != VQB_OK) return rc;
    leaky_relu_bwd_kernel<<<gs_blocks(n / 8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(y), static_cast<const __nv_bfloat16*>(dy), static_cast<__nv_bfloat16*>(dx),
        n / 8);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_wavelet_fwd(const float* x, void* y, const float* filt, int N, int C, int H, int W, int Cpad, void* stream) {
    VQB_CHECK(x && y && filt && H % 2 == 0 && W % 2 == 0 && Cpad % 8 == 0 && Cpad >= 4 * C,
              "vqb_wavelet_fwd: bad arguments (H, W even; Cpad >= 4C, multiple of 8)");
    const int64_t total = static_cast<int64_t>(N) * (H / 2) * (W / 2);
    wavelet_fwd_kernel<float><<<gs_blocks(total, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<__nv_bfloat16*>(y), filt, N, C, H, W, Cpad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_wavelet_fwd_bf16(const void* x, void* y, const float* filt, int N, int C, int H, int W, int Cpad,
                         void* stream) {
    VQB_CHECK(x && y && filt && N > 0 && C > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && Cpad % 8 == 0 &&
                  Cpad >= 4 * C,
              "vqb_wavelet_fwd_bf16: bad arguments (H, W even; Cpad >= 4C, multiple of 8)");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_wavelet_fwd_bf16: current device is not sm_90");
    const int64_t total = static_cast<int64_t>(N) * (H / 2) * (W / 2);
    wavelet_fwd_kernel<__nv_bfloat16><<<gs_blocks(total, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), filt, N, C, H, W, Cpad);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// out[c] = sum over P pixels of x[p][c]  (bias gradient). out is overwritten.
int vqb_colsum(const void* x, float* out, int64_t P, int C, void* stream) {
    VQB_CHECK(x && out && C % 8 == 0 && C <= 2048, "vqb_colsum: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    VQB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * C, st));
    const int V = C / 8, T = cv_threads(C), R = T / V;
    int bpsm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bpsm, colsum_kernel, T, C * sizeof(float)) != cudaSuccess || bpsm < 1)
        bpsm = 4;
    const int64_t concurrent = static_cast<int64_t>(num_sms() > 0 ? num_sms() : 132) * bpsm;
    int64_t nblk = concurrent;
    while (nblk < concurrent * 8 && (P + nblk - 1) / nblk > 2048) nblk += concurrent;
    int64_t ppc = (P + nblk - 1) / nblk;
    if (ppc < R * 4) ppc = R * 4;
    ppc = ((ppc + R - 1) / R) * R;
    const int chunks = static_cast<int>((P + ppc - 1) / ppc);
    colsum_kernel<<<chunks, T, C * sizeof(float), st>>>(static_cast<const __nv_bfloat16*>(x), out, P, C,
                                                        static_cast<int>(ppc));
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_wgrad_reduce(const float* partial, float* grad, int ksplit, int Cout, int CoutPad, int Cin, int T, int nslots,
                     int C64, const int* tapmap_dev, int accumulate, void* stream) {
    VQB_CHECK(partial && grad && tapmap_dev, "vqb_wgrad_reduce: null pointer");
    const int64_t total = static_cast<int64_t>(Cout) * Cin * T;
    wgrad_reduce_kernel<<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        partial, grad, ksplit, Cout, CoutPad, Cin, T, nslots, C64, tapmap_dev, accumulate);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_gauss_reparam(const void* z, const void* eps, void* out, int N, int Z, int64_t S, int bf16, void* stream) {
    VQB_CHECK(z && eps && out, "vqb_gauss_reparam: null pointer");
    VQB_CHECK(N > 0 && Z > 0 && S > 0 && (bf16 == 0 || bf16 == 1),
              "vqb_gauss_reparam: bad arguments (N=%d Z=%d S=%lld bf16=%d)", N, Z, (long long)S, bf16);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_gauss_reparam: current device is not sm_90");
    const int64_t total = static_cast<int64_t>(N) * Z * S;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (bf16)
        gauss_reparam_kernel<__nv_bfloat16><<<gs_blocks(total, 256), 256, 0, st>>>(
            static_cast<const __nv_bfloat16*>(z), static_cast<const __nv_bfloat16*>(eps),
            static_cast<__nv_bfloat16*>(out), Z, S, total);
    else
        gauss_reparam_kernel<float><<<gs_blocks(total, 256), 256, 0, st>>>(
            static_cast<const float*>(z), static_cast<const float*>(eps), static_cast<float*>(out), Z, S, total);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// tae.DiagonalGaussian backward (autograd of tae.py:263-264), see include/vqb200.h.
int vqb_gauss_reparam_bwd(const float* g, const float* z, const float* eps, float* dz, int N, int Z, int64_t S,
                          void* stream) {
    VQB_CHECK(g && z && eps && dz, "vqb_gauss_reparam_bwd: null pointer");
    VQB_CHECK(N > 0 && Z > 0 && S > 0, "vqb_gauss_reparam_bwd: bad arguments (N=%d Z=%d S=%lld)", N, Z, (long long)S);
    VQB_CHECK(((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(eps) |
                reinterpret_cast<uintptr_t>(dz)) & 3u) == 0,
              "vqb_gauss_reparam_bwd: pointers must be 4-byte aligned (fp32)");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_gauss_reparam_bwd: current device is not sm_90");
    const int64_t total = static_cast<int64_t>(N) * Z * S;
    gauss_reparam_bwd_kernel<<<gs_blocks(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(g, z, eps, dz, Z, S,
                                                                                                    total);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

}  // extern "C"
