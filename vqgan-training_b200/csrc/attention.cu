// Multi-head self-attention core of AttnBlock (ae.py:74-93): softmax(q k^T / sqrt(64)) v per head of 64 channels,
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
#include "common.cuh"
#include "ptx.cuh"

namespace vqb {

constexpr int kTQ = 64;   // rows per block (4 warps x 16)
constexpr int kLD = 72;   // smem row pitch in bf16 (144 B: conflict-free 32-bit fragment loads)

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 64 x COLS bf16 tile: rows row0.. of a [T][ld] matrix (column offset already applied to src) -> dst[64][kLD]; rows >= T
// zero.
template <int COLS = 64>
__device__ __forceinline__ void load_tile(__nv_bfloat16* dst, const __nv_bfloat16* src, int64_t ld, int row0, int T) {
    constexpr int kV = COLS / 8;  // 16-byte vectors per row
    for (int i = threadIdx.x; i < 64 * kV; i += blockDim.x) {
        const int r = i / kV, v = i % kV;
        uint4 u = make_uint4(0, 0, 0, 0);
        if (row0 + r < T) u = __ldg(reinterpret_cast<const uint4*>(src + static_cast<int64_t>(row0 + r) * ld + v * 8));
        *reinterpret_cast<uint4*>(dst + r * kLD + v * 8) = u;
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
// A fragments (16 rows of this warp x 16*KS cols) of a [64][kLD] smem tile
template <int KS = 4>
__device__ __forceinline__ void load_a_frags(const __nv_bfloat16* s, int warp, int lane, uint32_t (&a)[KS][4]) {
    const int r = warp * 16 + (lane >> 2), c = (lane & 3) * 2;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        a[ks][0] = *reinterpret_cast<const uint32_t*>(s + r * kLD + ks * 16 + c);
        a[ks][1] = *reinterpret_cast<const uint32_t*>(s + (r + 8) * kLD + ks * 16 + c);
        a[ks][2] = *reinterpret_cast<const uint32_t*>(s + r * kLD + ks * 16 + c + 8);
        a[ks][3] = *reinterpret_cast<const uint32_t*>(s + (r + 8) * kLD + ks * 16 + c + 8);
    }
}
// acc[nt] += A(16 x 16*KS) * B where B[k][n] = s[n][k] (s is a [8*NT n][kLD] smem tile, k contiguous)
template <int KS = 4, int NT = 8>
__device__ __forceinline__ void mma_a_bT(float (&acc)[NT][4], const uint32_t (&a)[KS][4], const __nv_bfloat16* s,
                                         int lane) {
    const int n = lane >> 2, c = (lane & 3) * 2;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const uint32_t b0 = *reinterpret_cast<const uint32_t*>(s + (nt * 8 + n) * kLD + ks * 16 + c);
            const uint32_t b1 = *reinterpret_cast<const uint32_t*>(s + (nt * 8 + n) * kLD + ks * 16 + c + 8);
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
// HD: head dim (64: ae.AttnBlock and tae heads of 64; 32: tae.AttnBlock at ch = 64). Q.K^T runs HD/16 k-steps over
// 8 key n-tiles; P.V runs 4 key k-steps over HD/8 output n-tiles.
template <int HD>
__global__ void __launch_bounds__(128) attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                       __nv_bfloat16* __restrict__ out, float* __restrict__ lse, int T,
                                                       int C, float scale) {
    constexpr int kKS = HD / 16, kNO = HD / 8;
    __shared__ __align__(16) __nv_bfloat16 sQ[64 * kLD];
    __shared__ __align__(16) __nv_bfloat16 sK[64 * kLD];
    __shared__ __align__(16) __nv_bfloat16 sVt[64 * kLD];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * kTQ, h = blockIdx.y, n = blockIdx.z, heads = gridDim.y;
    const int64_t ld = 3 * static_cast<int64_t>(C);
    const __nv_bfloat16* base = qkv + static_cast<int64_t>(n) * T * ld;
    load_tile<HD>(sQ, base + h * HD, ld, q0, T);
    __syncthreads();
    uint32_t qa[kKS][4];
    load_a_frags<kKS>(sQ, warp, lane, qa);
    float m_i[2] = {-INFINITY, -INFINITY}, l_i[2] = {0.f, 0.f};
    float o[kNO][4];
#pragma unroll
    for (int i = 0; i < kNO; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
    const int nkt = (T + 63) / 64;
    for (int kt = 0; kt < nkt; ++kt) {
        __syncthreads();
        load_tile<HD>(sK, base + C + h * HD, ld, kt * 64, T);
        load_tile_t<HD>(sVt, base + 2 * C + h * HD, ld, kt * 64, T);
        __syncthreads();
        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
        mma_a_bT<kKS, 8>(s, qa, sK, lane);
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

// D[n][h][q] = sum_d dO * O   (HD: head dim, 64 or 32; lane l holds channels 2l, 2l + 1 of the head)
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
    if (HD == 64 || lane * 2 < HD) {
        const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(o + off));
        const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + off));
        s = a.x * b.x + a.y * b.y;
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    if (lane == 0) {
        const int64_t n = nq / T, q = nq % T;
        dvec[(n * heads + h) * T + q] = s;
    }
}

// ------------------------------------------------------------------------------------------------ backward: dK, dV
// HD as in the forward: K.Q^T and V.dO^T run HD/16 k-steps over 8 query n-tiles; dV and dK run 4 query k-steps over HD/8
// n-tiles.
template <int HD>
__global__ void __launch_bounds__(128) attn_bwd_dkdv_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                            const __nv_bfloat16* __restrict__ dout,
                                                            const float* __restrict__ lse,
                                                            const float* __restrict__ dvec,
                                                            __nv_bfloat16* __restrict__ dqkv, int T, int C, float scale) {
    extern __shared__ __align__(16) uint8_t smem_dyn[];
    __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_dyn);
    __nv_bfloat16* sQt = sQ + 64 * kLD;
    __nv_bfloat16* sdO = sQt + 64 * kLD;
    __nv_bfloat16* sdOt = sdO + 64 * kLD;
    float* sLse = reinterpret_cast<float*>(sdOt + 64 * kLD);
    float* sD = sLse + 64;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k0 = blockIdx.x * 64, h = blockIdx.y, n = blockIdx.z, heads = gridDim.y;
    const int64_t ld = 3 * static_cast<int64_t>(C);
    const __nv_bfloat16* base = qkv + static_cast<int64_t>(n) * T * ld;
    constexpr int kKS = HD / 16, kNO = HD / 8;
    const __nv_bfloat16* dob = dout + static_cast<int64_t>(n) * T * C + h * HD;
    // K and V rows of this warp as A fragments (staged through sQ / sdO once)
    load_tile<HD>(sQ, base + C + h * HD, ld, k0, T);
    load_tile<HD>(sdO, base + 2 * C + h * HD, ld, k0, T);
    __syncthreads();
    uint32_t ka[kKS][4], va[kKS][4];
    load_a_frags<kKS>(sQ, warp, lane, ka);
    load_a_frags<kKS>(sdO, warp, lane, va);
    float dk[kNO][4], dv[kNO][4];
#pragma unroll
    for (int i = 0; i < kNO; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dk[i][j] = dv[i][j] = 0.f;
    const int key_r0 = k0 + warp * 16 + (lane >> 2);
    const int nqt = (T + 63) / 64;
    for (int qt = 0; qt < nqt; ++qt) {
        __syncthreads();
        load_tile<HD>(sQ, base + h * HD, ld, qt * 64, T);
        load_tile_t<HD>(sQt, base + h * HD, ld, qt * 64, T);
        load_tile<HD>(sdO, dob, C, qt * 64, T);
        load_tile_t<HD>(sdOt, dob, C, qt * 64, T);
        if (threadIdx.x < 64) {
            const int q = qt * 64 + threadIdx.x;
            sLse[threadIdx.x] = q < T ? lse[(static_cast<int64_t>(n) * heads + h) * T + q] : 0.f;
            sD[threadIdx.x] = q < T ? dvec[(static_cast<int64_t>(n) * heads + h) * T + q] : 0.f;
        }
        __syncthreads();
        float st[8][4], dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) st[i][j] = dp[i][j] = 0.f;
        mma_a_bT<kKS, 8>(st, ka, sQ, lane);   // S^T[key][q] = sum_d K[key][d] Q[q][d]
        mma_a_bT<kKS, 8>(dp, va, sdO, lane);  // dP^T[key][q] = sum_d V[key][d] dO[q][d]
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int ql = nt * 8 + (lane & 3) * 2 + (j & 1);
                const int key = key_r0 + (j >> 1) * 8;
                const bool ok = (qt * 64 + ql < T) && (key < T);
                const float pt = ok ? __expf(st[nt][j] * scale - sLse[ql]) : 0.f;
                st[nt][j] = pt;
                dp[nt][j] = pt * (dp[nt][j] - sD[ql]) * scale;
            }
        uint32_t pa[4][4], dsa[4][4];
        acc_to_a(st, pa);
        acc_to_a(dp, dsa);
        mma_a_bT<4, kNO>(dv, pa, sdOt, lane);  // dV[key][d] += sum_q P^T[key][q] dO[q][d]
        mma_a_bT<4, kNO>(dk, dsa, sQt, lane);  // dK[key][d] += sum_q dS^T[key][q] Q[q][d]
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int key = key_r0 + r * 8;
        if (key < T) {
            __nv_bfloat16* kp = dqkv + (static_cast<int64_t>(n) * T + key) * ld + C + h * HD + (lane & 3) * 2;
            __nv_bfloat16* vp = kp + C;
#pragma unroll
            for (int nt = 0; nt < kNO; ++nt) {
                *reinterpret_cast<uint32_t*>(kp + nt * 8) = pack_bf16x2(dk[nt][2 * r], dk[nt][2 * r + 1]);
                *reinterpret_cast<uint32_t*>(vp + nt * 8) = pack_bf16x2(dv[nt][2 * r], dv[nt][2 * r + 1]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward: dQ
// min-blocks 1 for heads of 32: without it ptxas caps the registers low and spills; heads of 64 keep the default
template <int HD>
__global__ void __launch_bounds__(128, HD == 32 ? 1 : 0) attn_bwd_dq_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                          const __nv_bfloat16* __restrict__ dout,
                                                          const float* __restrict__ lse, const float* __restrict__ dvec,
                                                          __nv_bfloat16* __restrict__ dqkv, int T, int C, float scale) {
    __shared__ __align__(16) __nv_bfloat16 sK[64 * kLD];
    __shared__ __align__(16) __nv_bfloat16 sKt[64 * kLD];
    __shared__ __align__(16) __nv_bfloat16 sV[64 * kLD];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * 64, h = blockIdx.y, n = blockIdx.z, heads = gridDim.y;
    const int64_t ld = 3 * static_cast<int64_t>(C);
    const __nv_bfloat16* base = qkv + static_cast<int64_t>(n) * T * ld;
    constexpr int kKS = HD / 16, kNO = HD / 8;
    const __nv_bfloat16* dob = dout + static_cast<int64_t>(n) * T * C + h * HD;
    load_tile<HD>(sK, base + h * HD, ld, q0, T);
    load_tile<HD>(sV, dob, C, q0, T);
    __syncthreads();
    uint32_t qa[kKS][4], doa[kKS][4];
    load_a_frags<kKS>(sK, warp, lane, qa);
    load_a_frags<kKS>(sV, warp, lane, doa);
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
        load_tile<HD>(sK, base + C + h * HD, ld, kt * 64, T);
        load_tile_t<HD>(sKt, base + C + h * HD, ld, kt * 64, T);
        load_tile<HD>(sV, base + 2 * C + h * HD, ld, kt * 64, T);
        __syncthreads();
        float s[8][4], dp[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
        mma_a_bT<kKS, 8>(s, qa, sK, lane);    // S[q][key]
        mma_a_bT<kKS, 8>(dp, doa, sV, lane);  // dP[q][key] = sum_d dO[q][d] V[key][d]
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
static int launch_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec,
                           void* dqkv, int N, int T, int C, float scale, cudaStream_t st) {
    const int heads = C / HD;
    const int64_t total = static_cast<int64_t>(N) * T * heads;
    attn_bwd_prep_kernel<HD><<<static_cast<int>((total + 7) / 8), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), dvec, T, C, heads, total);
    dim3 grid((T + 63) / 64, heads, N);
    const size_t smem = 4 * 64 * kLD * sizeof(__nv_bfloat16) + 2 * 64 * sizeof(float);
    static bool attr = false;
    if (!attr) {
        VQB_CUDA(cudaFuncSetAttribute(attn_bwd_dkdv_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      64 * 1024));
        attr = true;
    }
    attn_bwd_dkdv_kernel<HD><<<grid, 128, smem, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                       static_cast<const __nv_bfloat16*>(dout), lse, dvec,
                                                       static_cast<__nv_bfloat16*>(dqkv), T, C, scale);
    attn_bwd_dq_kernel<HD><<<grid, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                 static_cast<const __nv_bfloat16*>(dout), lse, dvec,
                                                 static_cast<__nv_bfloat16*>(dqkv), T, C, scale);
    VQB_CUDA(cudaGetLastError());
    count_launch(3);
    return VQB_OK;
}

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

// tae.AttnBlock (tae.py:26-51): heads of head_dim = C/8 channels, SDPA's default scale 1/sqrt(head_dim). Replaces
// F.scaled_dot_product_attention + the einops rearranges at tae.py:31-50.
int vqb_attn_fwd_hd(const void* qkv, void* out, float* lse, int N, int T, int C, int head_dim, void* stream) {
    VQB_CHECK(qkv && out && lse, "vqb_attn_fwd_hd: null pointer");
    VQB_CHECK(head_dim == 32 || head_dim == 64,
              "vqb_attn_fwd_hd: head_dim=%d is not supported (heads of 32 or 64 channels only)", head_dim);
    VQB_CHECK(C > 0 && C % head_dim == 0 && T > 0 && N > 0,
              "vqb_attn_fwd_hd: C=%d must be a positive multiple of head_dim %d (T=%d N=%d)", C, head_dim, T, N);
    VQB_CHECK(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(lse) & 3u) == 0,
              "vqb_attn_fwd_hd: qkv / out must be 16-byte aligned");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_attn_fwd_hd: current device is not sm_90");
    dim3 grid((T + 63) / 64, C / head_dim, N);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (head_dim == 64)
        attn_fwd_kernel<64><<<grid, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                   static_cast<__nv_bfloat16*>(out), lse, T, C, 0.125f);
    else
        attn_fwd_kernel<32><<<grid, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(qkv),
                                                   static_cast<__nv_bfloat16*>(out), lse, T, C,
                                                   0.17677669529663687f);  // 1/sqrt(32)
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
    VQB_CHECK(head_dim == 32 || head_dim == 64,
              "vqb_attn_bwd_hd: head_dim=%d is not supported (heads of 32 or 64 channels only)", head_dim);
    VQB_CHECK(C > 0 && C % head_dim == 0 && T > 0 && N > 0,
              "vqb_attn_bwd_hd: C=%d must be a positive multiple of head_dim %d (T=%d N=%d)", C, head_dim, T, N);
    VQB_CHECK(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out) |
                reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(dqkv)) & 15u) == 0 &&
                  ((reinterpret_cast<uintptr_t>(lse) | reinterpret_cast<uintptr_t>(dvec)) & 3u) == 0,
              "vqb_attn_bwd_hd: qkv / out / dout / dqkv must be 16-byte aligned");
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_attn_bwd_hd: current device is not sm_90");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (head_dim == 64) return launch_attn_bwd<64>(qkv, out, dout, lse, dvec, dqkv, N, T, C, 0.125f, st);
    return launch_attn_bwd<32>(qkv, out, dout, lse, dvec, dqkv, N, T, C, 0.17677669529663687f, st);  // 1/sqrt(32)
}

}  // extern "C"
