// Multi-head self-attention core of AttnBlock (ae.py:74-93, heads of 64) and tae.AttnBlock (heads of 8 to 112 channels),
// flash-attention style (online softmax, no T x T matrix in HBM), warp-level tensor-core MMA
// (mma.sync.m16n8k16 bf16 -> fp32). The 1x1 qkv / proj_out convolutions and the GroupNorm around it run on the
// wgmma conv / GN kernels; this file is only the [T x T] part: T = (H/8)(W/8) = 1024 tokens at 256^2, 8 heads at
// C = 512, 4.3 GFLOP per image and block (SURVEY.md a6) — latency/occupancy bound, not worth a TMA/wgmma pipeline.
//
// Layout: qkv [N][T][3C] bf16 (channel blocks q | k | v; head h owns channels h*64..h*64+63 of each block, the
// "b (h d) x y -> b h (x y) d" rearrange of ae.py:79-89 is pure addressing), out [N][T][C] bf16, lse [N][heads][T] fp32.
//
// Backward: D = rowsum(dO * O); one kernel owns key tiles and produces dK, dV; one owns query tiles and produces dQ.
// Both recompute P from q, k and the saved log-sum-exp.
#include <cmath>

#include "common.cuh"
#include "ptx.cuh"

namespace vqb {

constexpr int kTQ = 64;   // rows per block (4 warps x 16)
constexpr int kLD = 72;   // smem row pitch in bf16 (144 B: conflict-free 32-bit fragment loads)

// A head of HD channels (a multiple of 8, at most 112) is padded to kHP = the next multiple of 16 for the k-steps of
// Q.K^T; the padding columns of the [64][kHP] tiles are zero-filled in shared memory, never read from global memory.
// Tiles up to 64 channels keep the 72-element pitch; wider ones take kHP + 8 (conflict-free 32-bit fragment loads for
// every multiple of 16). Transposed tiles ([d][64 tokens], pitch kLD) get HD rows, at least 64.
template <int HD>
struct HeadShape {
    static_assert(HD % 8 == 0 && HD >= 8 && HD <= 112, "heads of 8 to 112 channels in steps of 8");
    static constexpr int kHP = (HD + 15) / 16 * 16;
    static constexpr int kL = kHP <= 64 ? kLD : kHP + 8;
    static constexpr int kRT = HD > 64 ? HD : 64;
    static constexpr int kKS = kHP / 16, kNO = HD / 8;
    static constexpr bool kSplitKV = kHP > 64;  // dK and dV in separate CTAs (attn_bwd_dkdv_kernel)
};

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 64 x COLS bf16 tile: rows row0.. of a [T][ld] matrix (column offset already applied to src) -> dst[64][LD]; rows >= T
// zero. PCOLS > COLS: columns COLS..PCOLS-1 (one 16-byte vector) are zero-filled.
template <int COLS = 64, int LD = kLD, int PCOLS = COLS>
__device__ __forceinline__ void load_tile(__nv_bfloat16* dst, const __nv_bfloat16* src, int64_t ld, int row0, int T) {
    constexpr int kV = COLS / 8;  // 16-byte vectors per row
    for (int i = threadIdx.x; i < 64 * kV; i += blockDim.x) {
        const int r = i / kV, v = i % kV;
        uint4 u = make_uint4(0, 0, 0, 0);
        if (row0 + r < T) u = __ldg(reinterpret_cast<const uint4*>(src + static_cast<int64_t>(row0 + r) * ld + v * 8));
        *reinterpret_cast<uint4*>(dst + r * LD + v * 8) = u;
    }
    if constexpr (PCOLS > COLS) {
        static_assert(PCOLS == COLS + 8, "one padding vector per row");
        for (int r = threadIdx.x; r < 64; r += blockDim.x)
            *reinterpret_cast<uint4*>(dst + r * LD + COLS) = make_uint4(0, 0, 0, 0);
    }
}
// same tile stored transposed: dst[col][row]
template <int COLS = 64>
__device__ __forceinline__ void load_tile_t(__nv_bfloat16* dst, const __nv_bfloat16* src, int64_t ld, int row0, int T) {
    constexpr int kV = COLS / 8;
    for (int i = threadIdx.x; i < 64 * kV; i += blockDim.x) {
        const int r = i / kV, v = i % kV;
        uint4 u = make_uint4(0, 0, 0, 0);
        if (row0 + r < T) u = __ldg(reinterpret_cast<const uint4*>(src + static_cast<int64_t>(row0 + r) * ld + v * 8));
        const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[(v * 8 + j) * kLD + r] = e[j];
    }
}
// A fragments (16 rows of this warp x 16*KS cols) of a [64][LD] smem tile
template <int KS = 4, int LD = kLD>
__device__ __forceinline__ void load_a_frags(const __nv_bfloat16* s, int warp, int lane, uint32_t (&a)[KS][4]) {
    const int r = warp * 16 + (lane >> 2), c = (lane & 3) * 2;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        a[ks][0] = *reinterpret_cast<const uint32_t*>(s + r * LD + ks * 16 + c);
        a[ks][1] = *reinterpret_cast<const uint32_t*>(s + (r + 8) * LD + ks * 16 + c);
        a[ks][2] = *reinterpret_cast<const uint32_t*>(s + r * LD + ks * 16 + c + 8);
        a[ks][3] = *reinterpret_cast<const uint32_t*>(s + (r + 8) * LD + ks * 16 + c + 8);
    }
}
// acc[nt] += A(16 x 16*KS) * B where B[k][n] = s[n][k] (s is a [8*NT n][LD] smem tile, k contiguous)
template <int KS = 4, int NT = 8, int LD = kLD>
__device__ __forceinline__ void mma_a_bT(float (&acc)[NT][4], const uint32_t (&a)[KS][4], const __nv_bfloat16* s,
                                         int lane) {
    const int n = lane >> 2, c = (lane & 3) * 2;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const uint32_t b0 = *reinterpret_cast<const uint32_t*>(s + (nt * 8 + n) * LD + ks * 16 + c);
            const uint32_t b1 = *reinterpret_cast<const uint32_t*>(s + (nt * 8 + n) * LD + ks * 16 + c + 8);
            mma16816(acc[nt], a[ks], b0, b1);
        }
}
// accumulator (16 x 64 fp32, 8 n-tiles) -> bf16 A fragments over k = the 64 columns
__device__ __forceinline__ void acc_to_a(const float (&p)[8][4], uint32_t (&a)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        a[kk][0] = pack_bf16x2(p[2 * kk][0], p[2 * kk][1]);
        a[kk][1] = pack_bf16x2(p[2 * kk][2], p[2 * kk][3]);
        a[kk][2] = pack_bf16x2(p[2 * kk + 1][0], p[2 * kk + 1][1]);
        a[kk][3] = pack_bf16x2(p[2 * kk + 1][2], p[2 * kk + 1][3]);
    }
}

// ------------------------------------------------------------------------------------------------ forward
// HD: head dim (64: ae.AttnBlock; tae.AttnBlock heads of C/8, any multiple of 8 up to 112). Q.K^T runs kHP/16 k-steps
// over 8 key n-tiles; P.V runs 4 key k-steps over HD/8 output n-tiles. Shared memory is static: 46,848 B at HD = 112.
// min-blocks 1 for heads of 72: without it ptxas caps the registers at 128 and spills
template <int HD>
__global__ void __launch_bounds__(128, HD == 72 ? 1 : 0) attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                       __nv_bfloat16* __restrict__ out, float* __restrict__ lse, int T,
                                                       int C, float scale) {
    using S = HeadShape<HD>;
    constexpr int kHP = S::kHP, kL = S::kL, kKS = S::kKS, kNO = S::kNO;
    __shared__ __align__(16) __nv_bfloat16 sQ[64 * kL];
    __shared__ __align__(16) __nv_bfloat16 sK[64 * kL];
    __shared__ __align__(16) __nv_bfloat16 sVt[S::kRT * kLD];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * kTQ, h = blockIdx.y, n = blockIdx.z, heads = gridDim.y;
    const int64_t ld = 3 * static_cast<int64_t>(C);
    const __nv_bfloat16* base = qkv + static_cast<int64_t>(n) * T * ld;
    load_tile<HD, kL, kHP>(sQ, base + h * HD, ld, q0, T);
    __syncthreads();
    uint32_t qa[kKS][4];
    load_a_frags<kKS, kL>(sQ, warp, lane, qa);
    float m_i[2] = {-INFINITY, -INFINITY}, l_i[2] = {0.f, 0.f};
    float o[kNO][4];
#pragma unroll
    for (int i = 0; i < kNO; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
    const int nkt = (T + 63) / 64;
    for (int kt = 0; kt < nkt; ++kt) {
        __syncthreads();
        load_tile<HD, kL, kHP>(sK, base + C + h * HD, ld, kt * 64, T);
        load_tile_t<HD>(sVt, base + 2 * C + h * HD, ld, kt * 64, T);
        __syncthreads();
        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
        mma_a_bT<kKS, 8, kL>(s, qa, sK, lane);
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int key = kt * 64 + nt * 8 + (lane & 3) * 2 + (j & 1);
                float v = s[nt][j] * scale;
                if (key >= T) v = -INFINITY;
                s[nt][j] = v;
                mx[j >> 1] = fmaxf(mx[j >> 1], v);
            }
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float mnew = fmaxf(m_i[r], mx[r]);
            alpha[r] = (m_i[r] == -INFINITY) ? 0.f : __expf(m_i[r] - mnew);
            m_i[r] = mnew;
        }
        float rs[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float pv = (s[nt][j] == -INFINITY) ? 0.f : __expf(s[nt][j] - m_i[j >> 1]);
                s[nt][j] = pv;
                rs[j >> 1] += pv;
            }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
            l_i[r] = l_i[r] * alpha[r] + rs[r];
        }
#pragma unroll
        for (int nt = 0; nt < kNO; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) o[nt][j] *= alpha[j >> 1];
        uint32_t pa[4][4];
        acc_to_a(s, pa);
        mma_a_bT<4, kNO>(o, pa, sVt, lane);  // B[k=key][n=d] = Vt[d][key]
    }
    const int r0 = q0 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = r0 + r * 8;
        if (q < T) {
            const float inv = 1.f / l_i[r];
            __nv_bfloat16* op = out + (static_cast<int64_t>(n) * T + q) * C + h * HD + (lane & 3) * 2;
#pragma unroll
            for (int nt = 0; nt < kNO; ++nt)
                *reinterpret_cast<uint32_t*>(op + nt * 8) = pack_bf16x2(o[nt][2 * r] * inv, o[nt][2 * r + 1] * inv);
            if ((lane & 3) == 0) lse[(static_cast<int64_t>(n) * heads + h) * T + q] = m_i[r] + __logf(l_i[r]);
        }
    }
}

// D[n][h][q] = sum_d dO * O   (HD: head dim; lane l holds channels 2l, 2l + 1 of the head, and 64 + 2l, 65 + 2l above
// 64)
template <int HD>
__global__ void attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout,
                                     float* __restrict__ dvec, int T, int C, int heads, int64_t total) {
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x / 32) + (threadIdx.x >> 5);  // one warp per (n,q,h)
    if (i >= total) return;
    const int lane = threadIdx.x & 31;
    const int h = static_cast<int>(i % heads);
    const int64_t nq = i / heads;
    const int64_t off = nq * C + h * HD + lane * 2;
    float s = 0.f;
    if (HD >= 64 || lane * 2 < HD) {
        const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(o + off));
        const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + off));
        s = a.x * b.x + a.y * b.y;
    }
    if constexpr (HD > 64) {
        if (64 + lane * 2 < HD) {
            const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(o + off + 64));
            const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + off + 64));
            s += a.x * b.x + a.y * b.y;
        }
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    if (lane == 0) {
        const int64_t n = nq / T, q = nq % T;
        dvec[(n * heads + h) * T + q] = s;
    }
}

// ------------------------------------------------------------------------------------------------ backward: dK, dV
// HD as in the forward: K.Q^T and V.dO^T run kHP/16 k-steps over 8 query n-tiles; dV and dK run 4 query k-steps over
// HD/8 n-tiles. kDK / kDV: which of dK, dV this CTA produces (both for heads up to 64 channels).
template <int HD, bool kDK, bool kDV>
__device__ __forceinline__ void attn_bwd_kv_tile(const __nv_bfloat16* __restrict__ qkv,
                                                 const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
                                                 const float* __restrict__ dvec, __nv_bfloat16* __restrict__ dqkv,
                                                 int T, int C, float scale, int h, int heads) {
    using S = HeadShape<HD>;
    constexpr int kHP = S::kHP, kL = S::kL, kKS = S::kKS, kNO = S::kNO;
    extern __shared__ __align__(16) uint8_t smem_dyn[];
    __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_dyn);
    __nv_bfloat16* sQt = sQ + 64 * kL;
    __nv_bfloat16* sdO = sQt + S::kRT * kLD;
    __nv_bfloat16* sdOt = sdO + 64 * kL;
    float* sLse = reinterpret_cast<float*>(sdOt + S::kRT * kLD);
    float* sD = sLse + 64;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k0 = blockIdx.x * 64, n = blockIdx.z;
    const int64_t ld = 3 * static_cast<int64_t>(C);
    const __nv_bfloat16* base = qkv + static_cast<int64_t>(n) * T * ld;
    const __nv_bfloat16* dob = dout + static_cast<int64_t>(n) * T * C + h * HD;
    // K and V rows of this warp as A fragments (staged through sQ / sdO once)
    load_tile<HD, kL, kHP>(sQ, base + C + h * HD, ld, k0, T);
    if constexpr (kDK) load_tile<HD, kL, kHP>(sdO, base + 2 * C + h * HD, ld, k0, T);
    __syncthreads();
    uint32_t ka[kKS][4], va[kKS][4];
    load_a_frags<kKS, kL>(sQ, warp, lane, ka);
    if constexpr (kDK) load_a_frags<kKS, kL>(sdO, warp, lane, va);
    float dk[kNO][4], dv[kNO][4];
#pragma unroll
    for (int i = 0; i < kNO; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dk[i][j] = dv[i][j] = 0.f;
    const int key_r0 = k0 + warp * 16 + (lane >> 2);
    const int nqt = (T + 63) / 64;
    for (int qt = 0; qt < nqt; ++qt) {
        __syncthreads();
        load_tile<HD, kL, kHP>(sQ, base + h * HD, ld, qt * 64, T);
        if constexpr (kDK) load_tile_t<HD>(sQt, base + h * HD, ld, qt * 64, T);
        if constexpr (kDK) load_tile<HD, kL, kHP>(sdO, dob, C, qt * 64, T);
        if constexpr (kDV) load_tile_t<HD>(sdOt, dob, C, qt * 64, T);
        if (threadIdx.x < 64) {
            const int q = qt * 64 + threadIdx.x;
            sLse[threadIdx.x] = q < T ? lse[(static_cast<int64_t>(n) * heads + h) * T + q] : 0.f;
            if constexpr (kDK) sD[threadIdx.x] = q < T ? dvec[(static_cast<int64_t>(n) * heads + h) * T + q] : 0.f;
        }
        __syncthreads();
        float st[8][4], dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) st[i][j] = dp[i][j] = 0.f;
        mma_a_bT<kKS, 8, kL>(st, ka, sQ, lane);                     // S^T[key][q] = sum_d K[key][d] Q[q][d]
        if constexpr (kDK) mma_a_bT<kKS, 8, kL>(dp, va, sdO, lane);  // dP^T[key][q] = sum_d V[key][d] dO[q][d]
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int ql = nt * 8 + (lane & 3) * 2 + (j & 1);
                const int key = key_r0 + (j >> 1) * 8;
                const bool ok = (qt * 64 + ql < T) && (key < T);
                const float pt = ok ? __expf(st[nt][j] * scale - sLse[ql]) : 0.f;
                st[nt][j] = pt;
                if constexpr (kDK) dp[nt][j] = pt * (dp[nt][j] - sD[ql]) * scale;
            }
        uint32_t pa[4][4], dsa[4][4];
        if constexpr (kDV) acc_to_a(st, pa);
        if constexpr (kDK) acc_to_a(dp, dsa);
        if constexpr (kDV) mma_a_bT<4, kNO>(dv, pa, sdOt, lane);  // dV[key][d] += sum_q P^T[key][q] dO[q][d]
        if constexpr (kDK) mma_a_bT<4, kNO>(dk, dsa, sQt, lane);  // dK[key][d] += sum_q dS^T[key][q] Q[q][d]
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int key = key_r0 + r * 8;
        if (key < T) {
            __nv_bfloat16* kp = dqkv + (static_cast<int64_t>(n) * T + key) * ld + C + h * HD + (lane & 3) * 2;
            __nv_bfloat16* vp = kp + C;
#pragma unroll
            for (int nt = 0; nt < kNO; ++nt) {
                if constexpr (kDK)
                    *reinterpret_cast<uint32_t*>(kp + nt * 8) = pack_bf16x2(dk[nt][2 * r], dk[nt][2 * r + 1]);
                if constexpr (kDV)
                    *reinterpret_cast<uint32_t*>(vp + nt * 8) = pack_bf16x2(dv[nt][2 * r], dv[nt][2 * r + 1]);
            }
        }
    }
}

// Heads up to 64 channels: one CTA per (key tile, head) produces dK and dV. Wider heads would hold K and V A fragments
// plus both accumulators (~260 registers at 112) and spill, so the work is split: blockIdx.y = 2 h + 1 produces dK,
// 2 h produces dV and recomputes S on its own (one more K.Q^T per tile, no dP, half the live accumulators).
// min-blocks 1 for heads of 56, which otherwise spill at a 168-register cap.
template <int HD>
__global__ void __launch_bounds__(128, HD == 56 ? 1 : 0) attn_bwd_dkdv_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                            const __nv_bfloat16* __restrict__ dout,
                                                            const float* __restrict__ lse,
                                                            const float* __restrict__ dvec,
                                                            __nv_bfloat16* __restrict__ dqkv, int T, int C, float scale) {
    if constexpr (!HeadShape<HD>::kSplitKV) {
        attn_bwd_kv_tile<HD, true, true>(qkv, dout, lse, dvec, dqkv, T, C, scale, blockIdx.y, gridDim.y);
    } else {
        const int h = blockIdx.y >> 1, heads = gridDim.y >> 1;
        if (blockIdx.y & 1)
            attn_bwd_kv_tile<HD, true, false>(qkv, dout, lse, dvec, dqkv, T, C, scale, h, heads);
        else
            attn_bwd_kv_tile<HD, false, true>(qkv, dout, lse, dvec, dqkv, T, C, scale, h, heads);
    }
}

// ------------------------------------------------------------------------------------------------ backward: dQ
// min-blocks 1 for heads of 32: without it ptxas caps the registers low and spills; heads of 64 keep the default
template <int HD>
__global__ void __launch_bounds__(128, HD == 32 ? 1 : 0) attn_bwd_dq_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                          const __nv_bfloat16* __restrict__ dout,
                                                          const float* __restrict__ lse, const float* __restrict__ dvec,
                                                          __nv_bfloat16* __restrict__ dqkv, int T, int C, float scale) {
    using S = HeadShape<HD>;
    constexpr int kHP = S::kHP, kL = S::kL, kKS = S::kKS, kNO = S::kNO;
    __shared__ __align__(16) __nv_bfloat16 sK[64 * kL];
    __shared__ __align__(16) __nv_bfloat16 sKt[S::kRT * kLD];
    __shared__ __align__(16) __nv_bfloat16 sV[64 * kL];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * 64, h = blockIdx.y, n = blockIdx.z, heads = gridDim.y;
    const int64_t ld = 3 * static_cast<int64_t>(C);
    const __nv_bfloat16* base = qkv + static_cast<int64_t>(n) * T * ld;
    const __nv_bfloat16* dob = dout + static_cast<int64_t>(n) * T * C + h * HD;
    load_tile<HD, kL, kHP>(sK, base + h * HD, ld, q0, T);
    load_tile<HD, kL, kHP>(sV, dob, C, q0, T);
    __syncthreads();
    uint32_t qa[kKS][4], doa[kKS][4];
    load_a_frags<kKS, kL>(sK, warp, lane, qa);
    load_a_frags<kKS, kL>(sV, warp, lane, doa);
    const int qr0 = q0 + warp * 16 + (lane >> 2);
    float lse_r[2], d_r[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = qr0 + r * 8;
        lse_r[r] = q < T ? lse[(static_cast<int64_t>(n) * heads + h) * T + q] : 0.f;
        d_r[r] = q < T ? dvec[(static_cast<int64_t>(n) * heads + h) * T + q] : 0.f;
    }
    float dq[kNO][4];
#pragma unroll
    for (int i = 0; i < kNO; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dq[i][j] = 0.f;
    const int nkt = (T + 63) / 64;
    for (int kt = 0; kt < nkt; ++kt) {
        __syncthreads();
        load_tile<HD, kL, kHP>(sK, base + C + h * HD, ld, kt * 64, T);
        load_tile_t<HD>(sKt, base + C + h * HD, ld, kt * 64, T);
        load_tile<HD, kL, kHP>(sV, base + 2 * C + h * HD, ld, kt * 64, T);
        __syncthreads();
        float s[8][4], dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
        mma_a_bT<kKS, 8, kL>(s, qa, sK, lane);    // S[q][key]
        mma_a_bT<kKS, 8, kL>(dp, doa, sV, lane);  // dP[q][key] = sum_d dO[q][d] V[key][d]
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int key = kt * 64 + nt * 8 + (lane & 3) * 2 + (j & 1);
                const int q = qr0 + (j >> 1) * 8;
                const bool ok = (key < T) && (q < T);
                const float pv = ok ? __expf(s[nt][j] * scale - lse_r[j >> 1]) : 0.f;
                dp[nt][j] = pv * (dp[nt][j] - d_r[j >> 1]) * scale;
            }
        uint32_t dsa[4][4];
        acc_to_a(dp, dsa);
        mma_a_bT<4, kNO>(dq, dsa, sKt, lane);  // dQ[q][d] += sum_key dS[q][key] K[key][d]
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = qr0 + r * 8;
        if (q < T) {
            __nv_bfloat16* qp = dqkv + (static_cast<int64_t>(n) * T + q) * ld + h * HD + (lane & 3) * 2;
#pragma unroll
            for (int nt = 0; nt < kNO; ++nt)
                *reinterpret_cast<uint32_t*>(qp + nt * 8) = pack_bf16x2(dq[nt][2 * r], dq[nt][2 * r + 1]);
        }
    }
}

template <int HD>
static void launch_attn_fwd(const void* qkv, void* out, float* lse, int N, int T, int C, float scale, cudaStream_t st) {
    dim3 grid((T + 63) / 64, C / HD, N);
    attn_fwd_kernel<HD><<<grid, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(out),
                                              lse, T, C, scale);
}

template <int HD>
static int launch_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec,
                           void* dqkv, int N, int T, int C, float scale, cudaStream_t st) {
    using S = HeadShape<HD>;
    const int heads = C / HD;
    const int64_t total = static_cast<int64_t>(N) * T * heads;
    attn_bwd_prep_kernel<HD><<<static_cast<int>((total + 7) / 8), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), dvec, T, C, heads, total);
    dim3 grid((T + 63) / 64, heads, N);
    dim3 grid_kv((T + 63) / 64, S::kSplitKV ? 2 * heads : heads, N);
    // sQ, sdO [64][kL]; sQt, sdOt [kRT][kLD]; lse, D: 63,488 B at HD = 112
    const size_t smem = (2 * 64 * S::kL + 2 * S::kRT * kLD) * sizeof(__nv_bfloat16) + 2 * 64 * sizeof(float);
    static bool attr = false;
    if (!attr) {
        VQB_CUDA(cudaFuncSetAttribute(attn_bwd_dkdv_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
        attr = true;
    }
    attn_bwd_dkdv_kernel<HD><<<grid_kv, 128, smem, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                          static_cast<const __nv_bfloat16*>(dout), lse, dvec,
                                                          static_cast<__nv_bfloat16*>(dqkv), T, C, scale);
    attn_bwd_dq_kernel<HD><<<grid, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                 static_cast<const __nv_bfloat16*>(dout), lse, dvec,
                                                 static_cast<__nv_bfloat16*>(dqkv), T, C, scale);
    VQB_CUDA(cudaGetLastError());
    count_launch(3);
    return VQB_OK;
}

// The head dimensions of vqb_attn_fwd_hd / vqb_attn_bwd_hd: multiples of 8 from 8 to 112 (tae.AttnBlock's C/8 for C a
// multiple of 64 up to 896).
#define VQB_ATTN_HEAD_DIMS(X) X(8) X(16) X(24) X(32) X(40) X(48) X(56) X(64) X(72) X(80) X(88) X(96) X(104) X(112)

static bool attn_head_dim_ok(int hd) { return hd >= 8 && hd <= 112 && hd % 8 == 0; }

// SDPA's default scale 1/sqrt(head_dim), rounded once to fp32 (0.125f at 64, 0.17677669529663687f at 32)
static float attn_scale(int hd) { return static_cast<float>(1.0 / std::sqrt(static_cast<double>(hd))); }

}  // namespace vqb

using namespace vqb;

extern "C" {

// out[n][t][h*64+d] = softmax_t'(q.k/8) v ; lse [N][C/64][T] saved for the backward. Replaces
// F.scaled_dot_product_attention + the einops rearranges at ae.py:79-89.
int vqb_attn_fwd(const void* qkv, void* out, float* lse, int N, int T, int C, void* stream) {
    VQB_CHECK(qkv && out && lse, "vqb_attn_fwd: null pointer");
    VQB_CHECK(C % 64 == 0 && T > 0 && N > 0, "vqb_attn_fwd: C=%d must be a multiple of the head dim 64", C);
    dim3 grid((T + 63) / 64, C / 64, N);
    attn_fwd_kernel<64><<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(out), lse, T, C, 0.125f);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// tae.AttnBlock (tae.py:26-51): heads of head_dim = C/8 channels (a multiple of 8 from 8 to 112), SDPA's default scale
// 1/sqrt(head_dim). Replaces F.scaled_dot_product_attention + the einops rearranges at tae.py:31-50.
int vqb_attn_fwd_hd(const void* qkv, void* out, float* lse, int N, int T, int C, int head_dim, void* stream) {
    VQB_CHECK(qkv && out && lse, "vqb_attn_fwd_hd: null pointer");
    VQB_CHECK(attn_head_dim_ok(head_dim),
              "vqb_attn_fwd_hd: head_dim=%d is not supported (heads of 8 to 112 channels in steps of 8 only)",
              head_dim);
    VQB_CHECK(C > 0 && C % head_dim == 0 && T > 0 && N > 0,
              "vqb_attn_fwd_hd: C=%d must be a positive multiple of head_dim %d (T=%d N=%d)", C, head_dim, T, N);
    VQB_CHECK(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(lse) & 3u) == 0,
              "vqb_attn_fwd_hd: qkv / out must be 16-byte aligned");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_attn_fwd_hd: current device is not sm_90");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (head_dim) {
#define VQB_ATTN_FWD_CASE(D) \
    case D: launch_attn_fwd<D>(qkv, out, lse, N, T, C, attn_scale(D), st); break;
        VQB_ATTN_HEAD_DIMS(VQB_ATTN_FWD_CASE)
#undef VQB_ATTN_FWD_CASE
    }
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// dqkv [N][T][3C] <- gradients of q, k, v. dvec: workspace [N][C/64][T] floats.
int vqb_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec, void* dqkv, int N,
                 int T, int C, void* stream) {
    VQB_CHECK(qkv && out && dout && lse && dvec && dqkv, "vqb_attn_bwd: null pointer");
    VQB_CHECK(C % 64 == 0 && T > 0 && N > 0, "vqb_attn_bwd: C=%d must be a multiple of the head dim 64", C);
    return launch_attn_bwd<64>(qkv, out, dout, lse, dvec, dqkv, N, T, C, 0.125f, static_cast<cudaStream_t>(stream));
}

// Backward of vqb_attn_fwd_hd (autograd of F.scaled_dot_product_attention at tae.py:31-50): heads of head_dim = C/8
// channels, scale 1/sqrt(head_dim). dqkv [N][T][3C]; dvec: workspace [N][C/head_dim][T] floats.
int vqb_attn_bwd_hd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec, void* dqkv,
                    int N, int T, int C, int head_dim, void* stream) {
    VQB_CHECK(qkv && out && dout && lse && dvec && dqkv, "vqb_attn_bwd_hd: null pointer");
    VQB_CHECK(attn_head_dim_ok(head_dim),
              "vqb_attn_bwd_hd: head_dim=%d is not supported (heads of 8 to 112 channels in steps of 8 only)",
              head_dim);
    VQB_CHECK(C > 0 && C % head_dim == 0 && T > 0 && N > 0,
              "vqb_attn_bwd_hd: C=%d must be a positive multiple of head_dim %d (T=%d N=%d)", C, head_dim, T, N);
    VQB_CHECK(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out) |
                reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(dqkv)) & 15u) == 0 &&
                  ((reinterpret_cast<uintptr_t>(lse) | reinterpret_cast<uintptr_t>(dvec)) & 3u) == 0,
              "vqb_attn_bwd_hd: qkv / out / dout / dqkv must be 16-byte aligned");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_attn_bwd_hd: current device is not sm_90");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (head_dim) {
#define VQB_ATTN_BWD_CASE(D) \
    case D: return launch_attn_bwd<D>(qkv, out, dout, lse, dvec, dqkv, N, T, C, attn_scale(D), st);
        VQB_ATTN_HEAD_DIMS(VQB_ATTN_BWD_CASE)
#undef VQB_ATTN_BWD_CASE
    }
    return VQB_OK;  // unreachable: head_dim was checked above
}

}  // extern "C"
