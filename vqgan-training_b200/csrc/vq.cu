// VQ codebook nearest-neighbour search (BASELINE.json config 4; absent from the reference — semantics pinned by
// oracle/vq_oracle.py): idx[i] = argmin_j sum_c (z[i][c] - e[j][c])^2 with the CANONICAL fp32 evaluation order
// (c ascending, separate rounded subtract / multiply / add, no FMA contraction) so that indices are bit-reproducible
// against the NumPy oracle; ties resolve to the smallest index (torch.argmin / np.argmin rule). Non-finite distances
// follow np.argmin too: the first NaN distance wins (a NaN in z[i] or in a code), and a row whose distances are all
// +inf (|z - e|^2 overflows) gets index 0, so the index is always in [0, K). Both the per-lane scan and the warp
// reduction compare the key (NaN -> -1, else d; distances are never negative) lexicographically with the index.
//
// One warp per row of z; the 32 lanes split the codebook (lane l scans codes l, l+32, ...), codebook chunks are staged
// in shared memory with a +1 word row pitch (conflict-free), the per-lane (distance, index) minima are combined with a
// lexicographic warp-shuffle reduction. HBM-light: z is read once, the 8192 x 16 fp32 codebook (512 KB) streams from L2.
#include "common.cuh"
#include "ptx.cuh"

namespace vqb {

constexpr int kVqRowsPerBlock = 32;  // 8 warps x 4 rows

__global__ void __launch_bounds__(256) vq_argmin_kernel(const float* __restrict__ z, const float* __restrict__ e,
                                                        long long* __restrict__ idx, float* __restrict__ zq,
                                                        float* __restrict__ sqerr, int M, int K, int D, int kVqChunk) {
    extern __shared__ float sm[];
    float* zs = sm;                             // [32][D]
    float* cs = sm + kVqRowsPerBlock * D;       // [chunk][D+1]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pitch = D + 1;
    for (int row0 = blockIdx.x * kVqRowsPerBlock; row0 < M; row0 += gridDim.x * kVqRowsPerBlock) {
        __syncthreads();
        for (int i = threadIdx.x; i < kVqRowsPerBlock * D; i += blockDim.x) {
            const int r = i / D;
            zs[i] = (row0 + r < M) ? z[static_cast<int64_t>(row0) * D + i] : 0.f;
        }
        float best_d[4];
        int best_j[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            best_d[r] = INFINITY;
            best_j[r] = 0x7fffffff;
        }
        for (int k0 = 0; k0 < K; k0 += kVqChunk) {
            const int nk = min(kVqChunk, K - k0);
            __syncthreads();
            for (int i = threadIdx.x; i < nk * D; i += blockDim.x) {
                const int j = i / D, c = i - j * D;
                cs[j * pitch + c] = e[static_cast<int64_t>(k0) * D + i];
            }
            __syncthreads();
            for (int j = lane; j < nk; j += 32) {
                const float* ej = cs + j * pitch;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const float* zr = zs + (warp * 4 + r) * D;
                    float d = 0.f;
                    for (int c = 0; c < D; ++c) {
                        const float diff = __fsub_rn(zr[c], ej[c]);
                        d = __fadd_rn(d, __fmul_rn(diff, diff));
                    }
                    // the first (smallest-index) minimum of this lane's subsequence wins; the index clause only takes
                    // the lane's first code when every key so far is +inf (the sentinel index is larger than any j)
                    const float key = d != d ? -1.f : d;
                    if (key < best_d[r] || (key == best_d[r] && k0 + j < best_j[r])) {
                        best_d[r] = key;
                        best_j[r] = k0 + j;
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            float d = best_d[r];
            int j = best_j[r];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float d2 = __shfl_xor_sync(0xffffffffu, d, o);
                const int j2 = __shfl_xor_sync(0xffffffffu, j, o);
                if (d2 < d || (d2 == d && j2 < j)) {
                    d = d2;
                    j = j2;
                }
            }
            const int row = row0 + warp * 4 + r;
            if (row < M) {
                if (lane == 0) idx[row] = j;
                float acc = 0.f;
                for (int c = lane; c < D; c += 32) {
                    const float q = e[static_cast<int64_t>(j) * D + c];
                    zq[static_cast<int64_t>(row) * D + c] = q;
                    const float df = q - zs[(warp * 4 + r) * D + c];
                    acc += df * df;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (lane == 0 && sqerr) atomicAdd(sqerr, acc);
            }
        }
    }
}

}  // namespace vqb

using namespace vqb;

extern "C" {

// z [M][D] fp32, codebook e [K][D] fp32 -> idx [M] int64, zq [M][D] = e[idx], *sqerr += sum (zq - z)^2 (optional).
int vqb_vq_argmin(const float* z, const float* e, long long* idx, float* zq, float* sqerr, int M, int K, int D,
                  void* stream) {
    VQB_CHECK(z && e && idx && zq, "vqb_vq_argmin: null pointer");
    VQB_CHECK(M > 0 && K > 0 && D > 0 && D <= 256, "vqb_vq_argmin: bad sizes M=%d K=%d D=%d", M, K, D);
    int kVqChunk = 1024;  // codes per shared-memory chunk (smaller for wide codes)
    while (kVqChunk > 32 && (static_cast<size_t>(kVqRowsPerBlock) * D + static_cast<size_t>(kVqChunk) * (D + 1)) * sizeof(float) > 160 * 1024)
        kVqChunk >>= 1;
    const size_t smem = (static_cast<size_t>(kVqRowsPerBlock) * D + static_cast<size_t>(kVqChunk) * (D + 1)) * sizeof(float);
    VQB_CHECK(smem <= 200 * 1024, "vqb_vq_argmin: D=%d too large for the shared-memory chunk", D);
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_vq_argmin: current device is not sm_90");
    static size_t attr_set = 0;
    if (smem > 48 * 1024 && smem > attr_set) {
        VQB_CUDA(cudaFuncSetAttribute(vq_argmin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set = 200 * 1024;
    }
    int blocks = (M + kVqRowsPerBlock - 1) / kVqRowsPerBlock;
    const int cap = (num_sms() > 0 ? num_sms() : 132) * 2;
    if (blocks > cap) blocks = cap;
    vq_argmin_kernel<<<blocks, 256, smem, static_cast<cudaStream_t>(stream)>>>(z, e, idx, zq, sqerr, M, K, D, kVqChunk);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

}  // extern "C"
