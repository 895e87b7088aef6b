// HBM-bound kernels of the LPIPS / VGG16 / PatchDiscriminator path.
//   max-pool 2x2 forward and (ReLU-masked) backward      torchvision vgg16.features[4,9,16,23]
//   LPIPS tail: channel-unit-normalise both feature maps, squared difference, 1x1 "lin" weights,
//   spatial mean -> per-image scalar; and its backward w.r.t. the reconstruction branch only
//   (the VGG trunk is frozen and the target branch carries no gradient).       utils.py:39-57,134-140
//
// One pass over the features per direction: the reference runs ~12 elementwise ATen kernels per layer
// (pow, sum, sqrt, add, div x2, sub, pow, conv1x1, mean) which re-read the 2 x 8 M elements/image each time.
#include "common.cuh"
#include "ptx.cuh"

namespace vqb {

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&f)[8]) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&f)[8]) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]);
    u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]);
    u.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(p) = u;
}

// ------------------------------------------------------------------ max-pool 2x2 stride 2
__global__ void maxpool2_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int Ho,
                                    int Wo, int C) {
    const int V = C >> 3;
    const int64_t total = static_cast<int64_t>(N) * Ho * Wo * V;
    const int W = 2 * Wo;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int cv = static_cast<int>(i % V);
        const int64_t pix = i / V;
        const int wo = static_cast<int>(pix % Wo);
        const int ho = static_cast<int>((pix / Wo) % Ho);
        const int64_t n = pix / (static_cast<int64_t>(Wo) * Ho);
        const __nv_bfloat16* s = x + ((n * 2 * Ho + 2 * ho) * W + 2 * wo) * C + cv * 8;
        float a[8], b[8], c[8], d[8];
        ld8(s, a);
        ld8(s + C, b);
        ld8(s + static_cast<int64_t>(W) * C, c);
        ld8(s + static_cast<int64_t>(W) * C + C, d);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = fmaxf(fmaxf(a[j], b[j]), fmaxf(c[j], d[j]));
        st8(y + pix * C + cv * 8, a);
    }
}

// dx[window] = dy at the FIRST maximal element of the window (PyTorch tie rule), zero elsewhere; if relu_mask the
// result is additionally gated by x > 0 (x is a post-ReLU activation: this is d(pre-activation)).
// `add` (optional, same shape as dx) is summed in: the LPIPS-tap / head gradient of the same node.
__global__ void maxpool2_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                    const __nv_bfloat16* __restrict__ add, __nv_bfloat16* __restrict__ dx, int N,
                                    int Ho, int Wo, int C, int relu_mask) {
    const int V = C >> 3;
    const int64_t total = static_cast<int64_t>(N) * Ho * Wo * V;
    const int W = 2 * Wo;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int cv = static_cast<int>(i % V);
        const int64_t pix = i / V;
        const int wo = static_cast<int>(pix % Wo);
        const int ho = static_cast<int>((pix / Wo) % Ho);
        const int64_t n = pix / (static_cast<int64_t>(Wo) * Ho);
        const int64_t o00 = ((n * 2 * Ho + 2 * ho) * W + 2 * wo) * C + cv * 8;
        const int64_t offs[4] = {o00, o00 + C, o00 + static_cast<int64_t>(W) * C, o00 + static_cast<int64_t>(W) * C + C};
        float v[4][8], g[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) ld8(x + offs[q], v[q]);
        ld8(dy + pix * C + cv * 8, g);
        float o[4][8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            int best = 0;
            float m = v[0][j];
#pragma unroll
            for (int q = 1; q < 4; ++q)
                if (v[q][j] > m) {
                    m = v[q][j];
                    best = q;
                }
            const float gg = (relu_mask && !(m > 0.f)) ? 0.f : g[j];
#pragma unroll
            for (int q = 0; q < 4; ++q) o[q][j] = (q == best) ? gg : 0.f;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (add) {
                float a[8];
                ld8(add + offs[q], a);
#pragma unroll
                for (int j = 0; j < 8; ++j) o[q][j] += a[j];
            }
            st8(dx + offs[q], o[q]);
        }
    }
}

// ------------------------------------------------------------------ LPIPS tail
// Train-mode dropout of NetLinLayer (utils.py:79-89: nn.Dropout(0.5) in front of the 1x1 lin conv; the reference never
// puts LPIPS in eval mode, vae_trainer.py:477): element (n, p, c) of the squared-difference tensor is kept with
// probability 1/2 and scaled by 2. The keep bit is a counter-based hash of (seed, flat NHWC element index) — the same
// function in forward, backward and vqb_lpips_dropout_mask (which materialises it for parity tests); 32 consecutive
// elements share one 64-bit mix (splitmix64 finaliser).
__device__ __forceinline__ uint32_t dropout_word(uint64_t seed, uint64_t word) {
    uint64_t z = seed + (word + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return static_cast<uint32_t>(z >> 32);
}
// keep bits of the 8 consecutive elements starting at flat index e0 (e0 % 8 == 0), bit j = element e0 + j
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, int64_t e0) {
    return (dropout_word(seed, static_cast<uint64_t>(e0) >> 5) >> (static_cast<uint32_t>(e0) & 31u)) & 0xFFu;
}

__global__ void lpips_dropout_mask_kernel(uint64_t seed, int64_t total8, uint8_t* __restrict__ mask) {
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total8;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const uint32_t k = dropout_keep8(seed, i * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j) mask[i * 8 + j] = (k >> j) & 1u;
    }
}

// A pixel is owned by G = min(32, C/8) lanes; each lane holds VPL = (C/8)/G 8-channel vectors of both features.
template <int VPL, bool DROP>
__global__ void lpips_tail_fwd_kernel(const __nv_bfloat16* __restrict__ f0, const __nv_bfloat16* __restrict__ f1,
                                      const float* __restrict__ w, float* __restrict__ out /* [N] */, int HW, int C,
                                      int G, int pix_per_block, float inv_hw, uint64_t seed) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int ppw = 32 / G;            // pixels per warp pass
    const int sub = lane / G;          // which pixel of the pass
    const int gl = lane % G;           // lane within the pixel group
    const int n = blockIdx.y;
    const int p0 = blockIdx.x * pix_per_block;
    const int p1 = min(HW, p0 + pix_per_block);
    float wreg[VPL][8];
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
        for (int j = 0; j < 8; ++j) wreg[v][j] = w[(gl + v * G) * 8 + j];
    float acc = 0.f;
    for (int pb = p0 + warp * ppw; pb < p1; pb += nwarps * ppw) {
        const int p = pb + sub;
        const bool ok = p < p1;
        float a[VPL][8], b[VPL][8];
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
            if (ok) {
                const int64_t off = (static_cast<int64_t>(n) * HW + p) * C + (gl + v * G) * 8;
                ld8(f0 + off, a[v]);
                ld8(f1 + off, b[v]);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) a[v][j] = b[v][j] = 0.f;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                s0 += a[v][j] * a[v][j];
                s1 += b[v][j] * b[v][j];
            }
        }
        for (int o = G >> 1; o > 0; o >>= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        }
        const float i0 = 1.f / (sqrtf(s0) + 1e-10f), i1 = 1.f / (sqrtf(s1) + 1e-10f);
        float d = 0.f;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
            uint32_t keep = 0xFFu;
            if (DROP) keep = dropout_keep8(seed, (static_cast<int64_t>(n) * HW + p) * C + (gl + v * G) * 8);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float t = a[v][j] * i0 - b[v][j] * i1;
                const float wj = DROP ? (((keep >> j) & 1u) ? 2.f * wreg[v][j] : 0.f) : wreg[v][j];
                d += wj * t * t;
            }
        }
        if (ok) acc += d;
    }
    // block reduction of acc
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ float red[32];
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        float t = lane < nwarps ? red[lane] : 0.f;
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) atomicAdd(&out[n], t * inv_hw);
    }
}

// d f0 = g[n]/HW * d val/d f0, gated by f0 > 0 (f0 is a post-ReLU VGG activation -> gradient of the pre-activation).
template <int VPL, bool DROP>
__global__ void lpips_tail_bwd_kernel(const __nv_bfloat16* __restrict__ f0, const __nv_bfloat16* __restrict__ f1,
                                      const float* __restrict__ w, const float* __restrict__ g /* [N] */,
                                      __nv_bfloat16* __restrict__ df0, int HW, int C, int G, int pix_per_block,
                                      float inv_hw, uint64_t seed) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int ppw = 32 / G, sub = lane / G, gl = lane % G;
    const int n = blockIdx.y;
    const int p0 = blockIdx.x * pix_per_block;
    const int p1 = min(HW, p0 + pix_per_block);
    const float gn = g[n] * inv_hw;
    float wreg[VPL][8];
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
        for (int j = 0; j < 8; ++j) wreg[v][j] = w[(gl + v * G) * 8 + j];
    for (int pb = p0 + warp * ppw; pb < p1; pb += nwarps * ppw) {
        const int p = pb + sub;
        const bool ok = p < p1;
        float a[VPL][8], b[VPL][8];
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
            if (ok) {
                const int64_t off = (static_cast<int64_t>(n) * HW + p) * C + (gl + v * G) * 8;
                ld8(f0 + off, a[v]);
                ld8(f1 + off, b[v]);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) a[v][j] = b[v][j] = 0.f;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                s0 += a[v][j] * a[v][j];
                s1 += b[v][j] * b[v][j];
            }
        }
        for (int o = G >> 1; o > 0; o >>= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        }
        const float nrm0 = sqrtf(s0);
        const float i0 = 1.f / (nrm0 + 1e-10f), i1 = 1.f / (sqrtf(s1) + 1e-10f);
        // q_c = 2 w_c (a_c i0 - b_c i1);  dot = sum_c q_c a_c
        float dot = 0.f;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
            uint32_t keep = 0xFFu;
            if (DROP) keep = dropout_keep8(seed, (static_cast<int64_t>(n) * HW + p) * C + (gl + v * G) * 8);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float wj = DROP ? (((keep >> j) & 1u) ? 2.f * wreg[v][j] : 0.f) : wreg[v][j];
                const float q = 2.f * wj * (a[v][j] * i0 - b[v][j] * i1);
                b[v][j] = q;  // reuse storage
                dot += q * a[v][j];
            }
        }
        for (int o = G >> 1; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        // d f0_k = q_k i0 - dot * f0_k * i0^2 / ||f0||      (second term defined as 0 when ||f0|| == 0)
        const float k2 = nrm0 > 0.f ? dot * i0 * i0 / nrm0 : 0.f;
        if (ok) {
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
                float o8[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float d = gn * (b[v][j] * i0 - k2 * a[v][j]);
                    o8[j] = a[v][j] > 0.f ? d : 0.f;
                }
                st8(df0 + (static_cast<int64_t>(n) * HW + p) * C + (gl + v * G) * 8, o8);
            }
        }
    }
}

static inline int gs_blocks2(int64_t total, int threads) {
    int64_t b = (total + threads - 1) / threads;
    const int64_t cap = static_cast<int64_t>(num_sms() > 0 ? num_sms() : 132) * 16;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return static_cast<int>(b);
}

}  // namespace vqb

using namespace vqb;

extern "C" {

int vqb_maxpool2_fwd(const void* x, void* y, int N, int Ho, int Wo, int C, void* stream) {
    VQB_CHECK(x && y && C % 8 == 0, "vqb_maxpool2_fwd: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * Ho * Wo * (C / 8);
    maxpool2_fwd_kernel<<<gs_blocks2(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), N, Ho, Wo, C);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_maxpool2_bwd(const void* x, const void* dy, const void* add, void* dx, int N, int Ho, int Wo, int C,
                     int relu_mask, void* stream) {
    VQB_CHECK(x && dy && dx && C % 8 == 0, "vqb_maxpool2_bwd: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * Ho * Wo * (C / 8);
    maxpool2_bwd_kernel<<<gs_blocks2(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(dy),
        static_cast<const __nv_bfloat16*>(add), static_cast<__nv_bfloat16*>(dx), N, Ho, Wo, C, relu_mask);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// Both directions serve exactly the widths whose C/8 channel vectors split over G = min(32, C/8) lanes (a power of two)
// of VPL = 1 or 2 vectors each: C = 64, 128, 256, 512. Sizes are checked before anything divides by them.
static int lpips_tail_check(const char* fn, int N, int HW, int C) {
    VQB_CHECK(N > 0 && HW > 0, "%s: bad sizes N=%d HW=%d", fn, N, HW);
    VQB_CHECK(C == 64 || C == 128 || C == 256 || C == 512, "%s: C=%d unsupported (64, 128, 256 or 512)", fn, C);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "%s: current device is not sm_90", fn);
    return VQB_OK;
}

// out[n] += (1/HW) sum_p sum_c w_c (f0/(|f0|+eps) - f1/(|f1|+eps))^2 ; out must be initialised by the caller
// (the five LPIPS layers accumulate into the same [N] vector, utils.py:54-57).
static int lpips_tail_fwd_impl(const char* fn, const void* f0, const void* f1, const float* w, float* out, int N,
                               int HW, int C, bool drop, uint64_t seed, void* stream) {
    VQB_CHECK(f0 && f1 && w && out, "%s: null pointer", fn);
    const int rc = lpips_tail_check(fn, N, HW, C);
    if (rc != VQB_OK) return rc;
    const int V = C / 8, G = V < 32 ? V : 32, VPL = V / G;
    int ppb = (HW + 132 * 4 - 1) / (132 * 4);
    const int per_pass = 8 * (32 / G);
    if (ppb < per_pass * 2) ppb = per_pass * 2;
    dim3 grid((HW + ppb - 1) / ppb, N);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float inv = 1.f / static_cast<float>(HW);
    const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(f0);
    const __nv_bfloat16* b = static_cast<const __nv_bfloat16*>(f1);
    if (VPL == 1 && !drop)
        lpips_tail_fwd_kernel<1, false><<<grid, 256, 0, st>>>(a, b, w, out, HW, C, G, ppb, inv, seed);
    else if (VPL == 2 && !drop)
        lpips_tail_fwd_kernel<2, false><<<grid, 256, 0, st>>>(a, b, w, out, HW, C, G, ppb, inv, seed);
    else if (VPL == 1)
        lpips_tail_fwd_kernel<1, true><<<grid, 256, 0, st>>>(a, b, w, out, HW, C, G, ppb, inv, seed);
    else if (VPL == 2)
        lpips_tail_fwd_kernel<2, true><<<grid, 256, 0, st>>>(a, b, w, out, HW, C, G, ppb, inv, seed);
    else
        return set_error(VQB_EINVAL, "%s: C=%d unsupported", fn, C);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_lpips_tail_fwd(const void* f0, const void* f1, const float* w, float* out, int N, int HW, int C, void* stream) {
    return lpips_tail_fwd_impl("vqb_lpips_tail_fwd", f0, f1, w, out, N, HW, C, false, 0, stream);
}
int vqb_lpips_tail_fwd_dropout(const void* f0, const void* f1, const float* w, float* out, int N, int HW, int C,
                               uint64_t seed, void* stream) {
    return lpips_tail_fwd_impl("vqb_lpips_tail_fwd_dropout", f0, f1, w, out, N, HW, C, true, seed, stream);
}
int vqb_lpips_dropout_mask(uint64_t seed, int N, int HW, int C, uint8_t* mask, void* stream) {
    VQB_CHECK(mask && N > 0 && HW > 0 && C > 0 && C % 8 == 0, "vqb_lpips_dropout_mask: bad arguments");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_lpips_dropout_mask: current device is not sm_90");
    const int64_t total8 = static_cast<int64_t>(N) * HW * C / 8;
    lpips_dropout_mask_kernel<<<gs_blocks2(total8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(seed, total8, mask);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

static int lpips_tail_bwd_impl(const char* fn, const void* f0, const void* f1, const float* w, const float* g,
                               void* df0, int N, int HW, int C, bool drop, uint64_t seed, void* stream) {
    VQB_CHECK(f0 && f1 && w && g && df0, "%s: null pointer", fn);
    const int rc = lpips_tail_check(fn, N, HW, C);
    if (rc != VQB_OK) return rc;
    const int V = C / 8, G = V < 32 ? V : 32, VPL = V / G;
    int ppb = (HW + 132 * 4 - 1) / (132 * 4);
    const int per_pass = 8 * (32 / G);
    if (ppb < per_pass * 2) ppb = per_pass * 2;
    dim3 grid((HW + ppb - 1) / ppb, N);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float inv = 1.f / static_cast<float>(HW);
    const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(f0);
    const __nv_bfloat16* b = static_cast<const __nv_bfloat16*>(f1);
    __nv_bfloat16* d = static_cast<__nv_bfloat16*>(df0);
    if (VPL == 1 && !drop)
        lpips_tail_bwd_kernel<1, false><<<grid, 256, 0, st>>>(a, b, w, g, d, HW, C, G, ppb, inv, seed);
    else if (VPL == 2 && !drop)
        lpips_tail_bwd_kernel<2, false><<<grid, 256, 0, st>>>(a, b, w, g, d, HW, C, G, ppb, inv, seed);
    else if (VPL == 1)
        lpips_tail_bwd_kernel<1, true><<<grid, 256, 0, st>>>(a, b, w, g, d, HW, C, G, ppb, inv, seed);
    else if (VPL == 2)
        lpips_tail_bwd_kernel<2, true><<<grid, 256, 0, st>>>(a, b, w, g, d, HW, C, G, ppb, inv, seed);
    else
        return set_error(VQB_EINVAL, "%s: C=%d unsupported", fn, C);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_lpips_tail_bwd(const void* f0, const void* f1, const float* w, const float* g, void* df0, int N, int HW, int C,
                       void* stream) {
    return lpips_tail_bwd_impl("vqb_lpips_tail_bwd", f0, f1, w, g, df0, N, HW, C, false, 0, stream);
}
int vqb_lpips_tail_bwd_dropout(const void* f0, const void* f1, const float* w, const float* g, void* df0, int N, int HW,
                               int C, uint64_t seed, void* stream) {
    return lpips_tail_bwd_impl("vqb_lpips_tail_bwd_dropout", f0, f1, w, g, df0, N, HW, C, true, seed, stream);
}

}  // extern "C"
