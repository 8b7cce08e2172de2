#include "host.h"

#include <stdlib.h>

#include <atomic>
#include <mutex>

#include "../../include/cogview_b200.h"

namespace cvh {

std::string& last_error() {
    static thread_local std::string s;
    return s;
}

int fail_arg(const char* fn, const char* msg) {
    last_error() = std::string(fn) + ": " + msg;
    return -1;
}
int fail_cuda(const char* fn, cudaError_t e) {
    last_error() = std::string(fn) + ": CUDA error " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return static_cast<int>(e);
}
int fail_cu(const char* fn, CUresult r) {
    last_error() = std::string(fn) + ": cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r);
    return -2;
}

static std::atomic<long long> g_launches{0};
void count_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launches() { return g_launches.load(std::memory_order_relaxed); }

bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("COGVIEW_B200_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

// SMs the persistent GEMM may occupy.  Under data parallelism the NCCL all-reduce kernels of the gradient buckets run
// concurrently with the backward GEMMs; a persistent grid sized to ALL SMs then finds a few of them taken and runs a
// second, nearly empty wave.  cv_set_reserved_sms(k) (or COGVIEW_B200_RESERVE_SMS) keeps k SMs free for them.
static std::atomic<int> g_reserved{-1};
int gemm_sms() {
    int r = g_reserved.load(std::memory_order_relaxed);
    if (r < 0) {
        const char* e = getenv("COGVIEW_B200_RESERVE_SMS");
        r = e ? atoi(e) : 0;
        if (r < 0) r = 0;
        g_reserved.store(r, std::memory_order_relaxed);
    }
    const int n = num_sms();
    return r < n - 8 ? n - r : 8;
}
void set_reserved_sms(int k) { g_reserved.store(k < 0 ? 0 : k, std::memory_order_relaxed); }

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
    });
    return fn;
}

int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, uint32_t rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides, Swizzle swz) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return fail_arg("encode_tmap", "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
    cuuint64_t gdim[5];
    cuuint64_t gstr[5];
    cuuint32_t bx[5];
    cuuint32_t es[5];
    for (uint32_t i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = elem_strides ? elem_strides[i] : 1;
        if (i + 1 < rank) gstr[i] = strides_bytes[i];
    }
    CUresult r = fn(out, dtype, rank, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swz == Swizzle::B128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail_cu("encode_tmap", r);
    return 0;
}

int encode_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                        uint32_t box_rows, uint32_t box_cols) {
    uint64_t dims[2] = {cols, rows};
    uint64_t str[1] = {ld * 2};
    uint32_t box[2] = {box_cols, box_rows};
    return encode_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, str, box, nullptr, Swizzle::B128);
}
int encode_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols) {
    uint64_t dims[2] = {cols, rows};
    uint64_t str[1] = {ld * 4};
    uint32_t box[2] = {box_cols, box_rows};
    return encode_tmap(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, str, box, nullptr, Swizzle::B128);
}

}  // namespace cvh

extern "C" {

const char* cv_last_error(void) { return cvh::last_error().c_str(); }

int cv_version(void) { return CV_B200_VERSION; }

long long cv_launch_count(void) { return cvh::launches(); }

int cv_set_reserved_sms(int k) {
    cvh::set_reserved_sms(k);
    return cvh::gemm_sms();
}

}
