// Optimizer-side kernels of the training step (HBM bound, one launch each per step):
//
//   vqb_adamw_flat          AdamW over ONE flat fp32 parameter/gradient/moment buffer holding every tensor of a model
//                           (two learning-rate groups + cosine schedule of vae_trainer.py:455-475,486-490 arrive as
//                           per-group scalars), replacing ~250 per-tensor ATen multi_tensor_apply chunks.
//   vqb_adamw_ema_flat_dev  the same AdamW pass that also moves an exponential moving average of the parameters (one
//                           more fp32 read and write per element, no extra launch).
//   vqb_pack_weights_multi  re-packs EVERY cached bf16 GEMM operand (forward, data-gradient, folded up-sample and
//                           fat-pixel layouts) of the just-updated fp32 OIHW master weights in one launch driven by a
//                           device-resident job table (what torch.autocast's per-step weight casts do in the reference,
//                           vae_trainer.py:453,623).
#include "common.cuh"
#include "ptx.cuh"

#include <cstring>

namespace vqb {

// ------------------------------------------------------------------ AdamW (decoupled weight decay; torch.optim.AdamW
// semantics incl. bias correction):  p *= 1 - lr*wd;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
//                                    p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
// The flat buffer is organised in 1024-element chunks; chunk_group[chunk] selects the hyper-parameter group (255 = the
// tensor owning this chunk received no gradient this step: skipped entirely, like torch skips `p.grad is None`).
struct AdamwGroups {
    float lr[VQB_ADAMW_MAX_GROUPS], beta1[VQB_ADAMW_MAX_GROUPS], beta2[VQB_ADAMW_MAX_GROUPS],
        eps[VQB_ADAMW_MAX_GROUPS], wd[VQB_ADAMW_MAX_GROUPS], bc1[VQB_ADAMW_MAX_GROUPS], bc2_sqrt[VQB_ADAMW_MAX_GROUPS];
};

// hyper-parameters either by value (h) or, hdev != nullptr, from DEVICE memory (one AdamwGroups record the host refreshes
// before every launch / CUDA-graph replay: learning-rate schedules and bias corrections then need no re-capture).
// kEma additionally keeps an exponential moving average of the parameters in the same pass over the chunks: after the
// AdamW update of a chunk (or, group 255, with its parameters unchanged) e -= r * (e - p'), r = 1 - d_n read from the
// device scalar ema_rate (vqb_adamw_ema_flat_dev). The AdamW arithmetic is the same code in both instances, so p, m and v
// are bit-identical with and without the average.
template <bool kEma>
__global__ void __launch_bounds__(256) adamw_flat_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                         float* __restrict__ m, float* __restrict__ v,
                                                         const uint8_t* __restrict__ chunk_group, int64_t nchunks,
                                                         AdamwGroups h, const AdamwGroups* __restrict__ hdev,
                                                         float grad_scale, float* __restrict__ ema,
                                                         const float* __restrict__ ema_rate) {
    if (hdev) h = *hdev;
    float rate = 0.f;
    if constexpr (kEma) rate = *ema_rate;
    for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const int grp = chunk_group[c];
        if (grp >= VQB_ADAMW_MAX_GROUPS) {
            if constexpr (kEma) {  // no gradient: AdamW skips the chunk, its average still moves toward the unchanged p
                const int64_t i = c * 1024 + threadIdx.x * 4;
                const float4 pp = *reinterpret_cast<const float4*>(p + i);
                float4 ee = *reinterpret_cast<const float4*>(ema + i);
                ee.x = ee.x - rate * (ee.x - pp.x);
                ee.y = ee.y - rate * (ee.y - pp.y);
                ee.z = ee.z - rate * (ee.z - pp.z);
                ee.w = ee.w - rate * (ee.w - pp.w);
                *reinterpret_cast<float4*>(ema + i) = ee;
            }
            continue;
        }
        const float lr = h.lr[grp], b1 = h.beta1[grp], b2 = h.beta2[grp], eps = h.eps[grp];
        const float decay = 1.f - lr * h.wd[grp], step = lr / h.bc1[grp], bc2s = h.bc2_sqrt[grp];
        const int64_t i = c * 1024 + threadIdx.x * 4;
        float4 pp = *reinterpret_cast<const float4*>(p + i);
        float4 gg = *reinterpret_cast<const float4*>(g + i);
        float4 mm = *reinterpret_cast<const float4*>(m + i);
        float4 vv = *reinterpret_cast<const float4*>(v + i);
        float* P = reinterpret_cast<float*>(&pp);
        float* G = reinterpret_cast<float*>(&gg);
        float* M = reinterpret_cast<float*>(&mm);
        float* V = reinterpret_cast<float*>(&vv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float gr = G[j] * grad_scale;
            float pj = P[j] * decay;
            M[j] = M[j] + (1.f - b1) * (gr - M[j]);          // lerp form, as ATen
            V[j] = b2 * V[j] + (1.f - b2) * gr * gr;
            const float denom = sqrtf(V[j]) / bc2s + eps;
            P[j] = pj - step * (M[j] / denom);
        }
        *reinterpret_cast<float4*>(p + i) = pp;
        *reinterpret_cast<float4*>(m + i) = mm;
        *reinterpret_cast<float4*>(v + i) = vv;
        if constexpr (kEma) {
            float4 ee = *reinterpret_cast<const float4*>(ema + i);
            float* E = reinterpret_cast<float*>(&ee);
#pragma unroll
            for (int j = 0; j < 4; ++j) E[j] = E[j] - rate * (E[j] - P[j]);
            *reinterpret_cast<float4*>(ema + i) = ee;
        }
    }
}

// ------------------------------------------------------------------ multi-tensor weight packing
// Each job packs one OIHW fp32 tensor into one bf16 operand:
//   out[r*ld_r + (slot / sg) * ld_g + (slot % sg) * Kpad + k] = bf16( transpose ? w[k][r][taps] : w[r][k][taps] ), k < K,
//   zero for K <= k < Kpad; `taps` = tapmap[slot] (one tap) or, fold = 1, the fp32 SUM over the taps whose bit is set.
// Normal layouts have sg = nslots (one group); the fat-pixel layout [R][3][64] has sg = 3, ld_g = 64 (columns beyond
// 3*Kpad stay at their initial zero). The master w is fp32 or (w_bf16 = 1, inference-only modules) bf16; either way the
// tile is staged in fp32, so a bf16 master is re-laid out exactly and folded taps are summed in fp32 before one rounding.
struct PackJob {
    const void* w;
    __nv_bfloat16* out;
    const int* tapmap;
    int Cout, Cin, T, nslots, transpose, Kpad, fold, sg, ld_g, ld_r;
    int first_block;  // prefix sum of ceil(R/8)*ceil(Kpad/64) tile blocks over the jobs before this one
    int w_bf16;
};

static_assert(sizeof(PackJob) == sizeof(VqbPackJob), "PackJob must mirror VqbPackJob");
constexpr int kPackRows = 8, kPackK = 64, kPackMaxT = 16;

// forward layout tile[r*64T + (k*T + t)], transposed tile[k*(8T+1) + (r*T + t)] (no runtime divisions)
template <typename Src>
__device__ __forceinline__ void pack_load_tile(const PackJob& jb, const Src* w, float* tile, int r0, int k0, int nr,
                                               int nk, int warp, int lane) {
    const int T = jb.T;
    if (!jb.transpose) {
        const int run = nk * T;  // contiguous elements of one row
        for (int r = warp; r < kPackRows; r += 8) {
            const Src* src = w + (static_cast<int64_t>(r0 + r) * jb.Cin + k0) * T;
            for (int e = lane; e < kPackK * T; e += 32)
                tile[r * kPackK * T + e] = (r < nr && e < run) ? to_f32(src[e]) : 0.f;
        }
    } else {
        const int run = nr * T;  // contiguous elements of one k (= one output channel's rows r0..r0+7)
        const int kstride = kPackRows * T + 1;
        for (int k = warp; k < kPackK; k += 8) {
            const Src* src = w + (static_cast<int64_t>(k0 + k) * jb.Cin + r0) * T;
            for (int e = lane; e < kPackRows * T; e += 32)
                tile[k * kstride + e] = (k < nk && e < run) ? to_f32(src[e]) : 0.f;
        }
    }
}

// One block = an (8 rows) x (64 k) tile of one job, all slots: the OIHW source is read in contiguous runs (64*T floats per
// row for the forward layout, 8*T floats per k for the transposed one) into shared memory, then every slot's 64
// consecutive bf16 (128 B) are written coalesced, so the re-pack streams HBM / L2 instead of reading with a stride of T
// floats.
__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const PackJob* __restrict__ jobs, int njobs) {
    __shared__ float tile[kPackK * (kPackRows * kPackMaxT + 1)];
    // binary search: last job with first_block <= blockIdx.x
    int lo = 0, hi = njobs - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (jobs[mid].first_block <= static_cast<int>(blockIdx.x)) lo = mid; else hi = mid - 1;
    }
    const PackJob jb = jobs[lo];
    const int R = jb.transpose ? jb.Cin : jb.Cout;
    const int K = jb.transpose ? jb.Cout : jb.Cin;
    const int T = jb.T;
    const int kblocks = (jb.Kpad + kPackK - 1) / kPackK;
    const int bid = static_cast<int>(blockIdx.x) - jb.first_block;
    const int r0 = (bid / kblocks) * kPackRows, k0 = (bid % kblocks) * kPackK;
    const int nr = min(kPackRows, R - r0), nk = max(0, min(kPackK, K - k0));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (jb.w_bf16)
        pack_load_tile(jb, static_cast<const __nv_bfloat16*>(jb.w), tile, r0, k0, nr, nk, warp, lane);
    else
        pack_load_tile(jb, static_cast<const float*>(jb.w), tile, r0, k0, nr, nk, warp, lane);
    __syncthreads();
    // ---- store: thread = (row pair q, k); every (row, slot) writes 64 consecutive bf16
    const int k = threadIdx.x & (kPackK - 1), q = threadIdx.x >> 6;
    if (k0 + k < jb.Kpad) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const int r = q * 2 + rr;
            if (r >= nr) break;
            const float* tp = jb.transpose ? tile + k * (kPackRows * T + 1) + r * T : tile + (r * kPackK + k) * T;
            __nv_bfloat16* orow = jb.out + static_cast<int64_t>(r0 + r) * jb.ld_r + k0 + k;
            int sl = 0, grp = 0;  // slot within its group, group index (no divisions)
            for (int slot = 0; slot < jb.nslots; ++slot) {
                const int tm = jb.tapmap[slot];
                float val = 0.f;
                if (jb.fold) {
                    for (int t = 0; t < T; ++t)
                        if ((tm >> t) & 1) val += tp[t];
                } else {
                    val = tp[tm];
                }
                orow[grp * jb.ld_g + sl * jb.Kpad] = __float2bfloat16(val);
                if (++sl == jb.sg) {
                    sl = 0;
                    ++grp;
                }
            }
        }
    }
}

}  // namespace vqb

using namespace vqb;

extern "C" {

int vqb_adamw_flat(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const uint8_t* chunk_group,
                   int64_t nchunks, int ngroups, const VqbAdamwGroup* groups_host, float grad_scale, void* stream) {
    VQB_CHECK(params && grads && exp_avg && exp_avg_sq && chunk_group && groups_host, "vqb_adamw_flat: null pointer");
    VQB_CHECK(ngroups >= 1 && ngroups <= VQB_ADAMW_MAX_GROUPS, "vqb_adamw_flat: ngroups %d out of range", ngroups);
    VQB_CHECK((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) |
               reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq)) % 16 == 0,
              "vqb_adamw_flat: buffers must be 16-byte aligned");
    if (nchunks <= 0) return VQB_OK;
    AdamwGroups h;
    for (int i = 0; i < VQB_ADAMW_MAX_GROUPS; ++i) {
        const VqbAdamwGroup& s = groups_host[i < ngroups ? i : 0];
        VQB_CHECK(s.step >= 1, "vqb_adamw_flat: step must be >= 1");
        h.lr[i] = s.lr; h.beta1[i] = s.beta1; h.beta2[i] = s.beta2; h.eps[i] = s.eps; h.wd[i] = s.weight_decay;
        // bias corrections in double, like torch's python-side computation
        h.bc1[i] = static_cast<float>(1.0 - pow(static_cast<double>(s.beta1), static_cast<double>(s.step)));
        h.bc2_sqrt[i] = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(s.beta2), static_cast<double>(s.step))));
    }
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_adamw_flat: current device is not sm_90");
    int64_t blocks = nchunks;
    const int64_t cap = static_cast<int64_t>(num_sms() > 0 ? num_sms() : 132) * 16;
    if (blocks > cap) blocks = cap;
    adamw_flat_kernel<false><<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        params, grads, exp_avg, exp_avg_sq, chunk_group, nchunks, h, nullptr, grad_scale, nullptr, nullptr);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

// Fills the 28-float device record of vqb_adamw_flat_dev from host-side group descriptions (host function: the caller
// copies `record_host` to the device, e.g. from pinned memory on the launch stream).
int vqb_adamw_fill_record(int ngroups, const VqbAdamwGroup* groups_host, float* record_host /* [28] */) {
    VQB_CHECK(groups_host && record_host && ngroups >= 1 && ngroups <= VQB_ADAMW_MAX_GROUPS,
              "vqb_adamw_fill_record: bad arguments");
    AdamwGroups h;
    for (int i = 0; i < VQB_ADAMW_MAX_GROUPS; ++i) {
        const VqbAdamwGroup& s = groups_host[i < ngroups ? i : 0];
        VQB_CHECK(s.step >= 1, "vqb_adamw_fill_record: step must be >= 1");
        h.lr[i] = s.lr; h.beta1[i] = s.beta1; h.beta2[i] = s.beta2; h.eps[i] = s.eps; h.wd[i] = s.weight_decay;
        h.bc1[i] = static_cast<float>(1.0 - pow(static_cast<double>(s.beta1), static_cast<double>(s.step)));
        h.bc2_sqrt[i] = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(s.beta2), static_cast<double>(s.step))));
    }
    static_assert(sizeof(AdamwGroups) == 28 * sizeof(float), "record layout");
    memcpy(record_host, &h, sizeof(h));
    return VQB_OK;
}

int vqb_adamw_flat_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const uint8_t* chunk_group,
                       int64_t nchunks, const float* record_dev, float grad_scale, void* stream) {
    VQB_CHECK(params && grads && exp_avg && exp_avg_sq && chunk_group && record_dev, "vqb_adamw_flat_dev: null pointer");
    VQB_CHECK((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) |
               reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq)) % 16 == 0,
              "vqb_adamw_flat_dev: buffers must be 16-byte aligned");
    if (nchunks <= 0) return VQB_OK;
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_adamw_flat_dev: current device is not sm_90");
    int64_t blocks = nchunks;
    const int64_t cap = static_cast<int64_t>(num_sms() > 0 ? num_sms() : 132) * 16;
    if (blocks > cap) blocks = cap;
    AdamwGroups dummy = {};
    adamw_flat_kernel<false><<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        params, grads, exp_avg, exp_avg_sq, chunk_group, nchunks, dummy,
        reinterpret_cast<const AdamwGroups*>(record_dev), grad_scale, nullptr, nullptr);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_adamw_ema_flat_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, float* ema,
                           const uint8_t* chunk_group, int64_t nchunks, const float* record_dev,
                           const float* ema_rate_dev, float grad_scale, void* stream) {
    VQB_CHECK(params && grads && exp_avg && exp_avg_sq && ema && chunk_group && record_dev && ema_rate_dev,
              "vqb_adamw_ema_flat_dev: null pointer");
    VQB_CHECK((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) |
               reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq) |
               reinterpret_cast<uintptr_t>(ema)) % 16 == 0,
              "vqb_adamw_ema_flat_dev: buffers must be 16-byte aligned");
    if (nchunks <= 0) return VQB_OK;
    if (!device_is_sm90()) return set_error(VQB_ENODEVICE, "vqb_adamw_ema_flat_dev: current device is not sm_90");
    int64_t blocks = nchunks;
    const int64_t cap = static_cast<int64_t>(num_sms() > 0 ? num_sms() : 132) * 16;
    if (blocks > cap) blocks = cap;
    AdamwGroups dummy = {};
    adamw_flat_kernel<true><<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        params, grads, exp_avg, exp_avg_sq, chunk_group, nchunks, dummy,
        reinterpret_cast<const AdamwGroups*>(record_dev), grad_scale, ema, ema_rate_dev);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

int vqb_pack_weights_multi(const VqbPackJob* jobs_dev, int njobs, int total_blocks, void* stream) {
    VQB_CHECK(jobs_dev && njobs >= 1 && total_blocks >= 1, "vqb_pack_weights_multi: bad arguments");  // (T <= 16 per job)
    pack_weights_multi_kernel<<<total_blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const PackJob*>(jobs_dev), njobs);
    VQB_CUDA(cudaGetLastError());
    count_launch();
    return VQB_OK;
}

}  // extern "C"
