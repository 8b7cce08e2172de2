// Host-side helpers shared by the C-ABI translation units: error reporting, TMA tensor-map
// encoding through the driver entry point (no link-time dependency on libcuda), launch checks.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace cvh {

// last-error string returned by cv_last_error() (thread-local: entry points are re-entrant)
std::string& last_error();
int fail_arg(const char* fn, const char* msg);          // returns a negative code (argument error)
int fail_cuda(const char* fn, cudaError_t e);           // returns the positive cudaError_t
int fail_cu(const char* fn, CUresult r);                // driver error while encoding a tensor map

#define CV_REQUIRE(cond, msg)                                  \
    do {                                                       \
        if (!(cond)) return cvh::fail_arg(__func__, msg);      \
    } while (0)

#define CV_CUDA(expr)                                          \
    do {                                                       \
        cudaError_t _e = (expr);                               \
        if (_e != cudaSuccess) return cvh::fail_cuda(__func__, _e); \
    } while (0)

#define CV_LAUNCH_CHECK()                                      \
    do {                                                       \
        cudaError_t _e = cudaGetLastError();                   \
        if (_e != cudaSuccess) return cvh::fail_cuda(__func__, _e); \
        cvh::count_launches(1);                                \
    } while (0)

// host-side description of a dropout site (see cv::DropoutArgs)
struct HostDropout {
    float p, scale;
    uint32_t threshold, stream;
    uint64_t seed;
};
inline HostDropout make_dropout(float p, uint64_t seed, uint32_t stream) {
    HostDropout d;
    d.p = p;
    d.scale = p > 0.f ? 1.0f / (1.0f - p) : 1.0f;
    double t = (double)p * 4294967296.0;
    d.threshold = t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
    d.stream = stream;
    d.seed = seed;
    return d;
}

int num_sms();
int gemm_sms();               // num_sms() minus the SMs reserved for concurrently running collectives
void set_reserved_sms(int k);
void count_launches(int n);
long long launches();   // kernels launched by this library since load (cv_launch_count)

// Launch with programmatic dependent launch (PDL) allowed: the kernel may become resident while the previous
// kernel in the stream drains.  Such kernels call cv::pdl_wait() before touching anything the previous kernel
// wrote.  COGVIEW_B200_PDL=0 disables the attribute (plain stream order).
bool pdl_enabled();
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                       Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (pdl && pdl_enabled()) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

enum class Swizzle { None, B128 };

// Encode a tiled tensor map.  dims/strides are innermost-first, strides in BYTES for dims 1..rank-1.
// elem_strides may be null (all ones).  Returns 0 or an error code (with last_error set).
int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, uint32_t rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides, Swizzle swz);

// 2-D row-major bf16 matrix [rows, cols] with leading dimension ld (elements); box = [box_rows, box_cols]
int encode_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                        uint32_t box_rows, uint32_t box_cols);
int encode_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols);

}  // namespace cvh
