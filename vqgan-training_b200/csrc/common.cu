#include "common.cuh"

#include <atomic>
#include <cstring>
#include <cudaTypedefs.h>
#include <mutex>

namespace vqb {

static thread_local char g_err[512] = "";
static std::atomic<int> g_launches{0};

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
        else
            (void)cudaGetLastError();
    });
    return fn;
}

int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box, int swizzle_bytes) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return set_error(VQB_ENODEVICE, "cuTensorMapEncodeTiled driver entry point unavailable");
    if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0)
        return set_error(VQB_EINVAL, "tensor map base %p not 16-byte aligned", base);
    cuuint64_t gdim[5];
    cuuint64_t gstr[4];
    cuuint32_t bx[5];
    cuuint32_t es[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
        if (box[i] == 0 || box[i] > 256) return set_error(VQB_EINVAL, "tensor map box[%d]=%u out of range", i, box[i]);
    }
    for (int i = 0; i + 1 < rank; ++i) {
        gstr[i] = strides_bytes[i];
        if (gstr[i] % 16 != 0) return set_error(VQB_EINVAL, "tensor map stride[%d]=%llu not a multiple of 16 B", i,
                                                (unsigned long long)gstr[i]);
    }
    CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
    if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
    if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
    if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                    gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT || r == CUDA_ERROR_NOT_INITIALIZED) {
        // first driver-API call on this host thread (e.g. an autograd worker whose first op is ours): the runtime binds
        // the primary context lazily, so force it and retry once
        cudaFree(nullptr);
        r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr,
               bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) {
        return set_error(VQB_ECUDA,
                         "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] box [%u %u %u %u] "
                         "stride0 %llu",
                         (int)r, rank, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0),
                         (unsigned long long)(rank > 2 ? gdim[2] : 0), (unsigned long long)(rank > 3 ? gdim[3] : 0),
                         bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0, rank > 3 ? bx[3] : 0,
                         (unsigned long long)(rank > 1 ? gstr[0] : 0));
    }
    return VQB_OK;
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 0;
    }
    return n;
}

bool device_is_sm90() {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        (void)cudaGetLastError();
        return false;
    }
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
        (void)cudaGetLastError();
        return false;
    }
    return major == 9;
}

}  // namespace vqb

extern "C" {

const char* vqb_last_error(void) { return vqb::g_err; }
int vqb_version(void) { return 103; }
int vqb_device_ok(void) { return (vqb::device_is_sm90() && vqb::get_encode_fn() != nullptr) ? 1 : 0; }
int vqb_kernel_launch_count(void) { return vqb::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
