// Host-side helpers shared by all translation units of libvqb200.so:
// error reporting, launch counting, TMA tensor-map encoding through the driver entry point.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_runtime.h>

#include "../../include/vqb200.h"

namespace vqb {

int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);

// Encodes a bf16 tiled tensor map (rank 2..5). dims/strides innermost-first; strides in BYTES for
// dims 1..rank-1 (dim 0 is contiguous). swizzle_bytes in {0,32,64,128}. Returns 0 or negative code.
int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box, int swizzle_bytes);

int num_sms();
bool device_is_sm90();

#define VQB_CHECK(cond, ...)                              \
    do {                                                  \
        if (!(cond)) return vqb::set_error(VQB_EINVAL, __VA_ARGS__); \
    } while (0)

#define VQB_CUDA(call)                                                                            \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess)                                                                   \
            return vqb::set_error(VQB_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                                  __FILE__, __LINE__);                                            \
    } while (0)

inline int ilog2(uint32_t v) {
    int l = 0;
    while ((1u << (l + 1)) <= v) ++l;
    return l;
}
inline uint32_t next_pow2(uint32_t v) {
    uint32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

}  // namespace vqb
