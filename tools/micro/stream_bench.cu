// Micro-benchmark: how fast can one persistent CTA per SM stream a big buffer through a shared-memory ring with
// cp.async.bulk row copies?  Variants: bytes per copy, smem row pitch, stages, consumer work.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o stream_bench stream_bench.cu && ./stream_bench
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t done = 0;
    while (!done)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol, int hint) {
    if (hint)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                     ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
    else
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

struct Cfg {
    int rows, row_bytes, pitch, nst, consumers, work, hint, src_stride;   // src_stride: bytes between source rows
    long long stages_per_cta;
};

__global__ void __launch_bounds__(544, 1) stream_kernel(const uint8_t* __restrict__ src, size_t src_bytes, Cfg c,
                                                        unsigned long long* out) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);
    uint64_t* empty = full + 16;
    const uint32_t ring = smem_u32(smem + 1024);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int stage_bytes = (c.rows * c.pitch + 127) / 128 * 128;
    if (tid == 0) {
        for (int i = 0; i < c.nst; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], c.consumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const size_t per_stage_src = (size_t)c.rows * c.src_stride;
    const size_t base = (size_t)blockIdx.x * c.stages_per_cta * per_stage_src;
    if (warp == 16) {
        uint64_t pol;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
        int st = 0; uint32_t ph = 0;
        for (long long i = 0; i < c.stages_per_cta; ++i) {
            mbar_wait(&empty[st], ph ^ 1);
            if (lane == 0) mbar_expect_tx(&full[st], c.rows * c.row_bytes);
            __syncwarp();
            const size_t o = (base + i * per_stage_src) % (src_bytes - per_stage_src);
            if (lane < c.rows)
                bulk_g2s(ring + st * stage_bytes + lane * c.pitch, src + (o & ~(size_t)127) + (size_t)lane * c.src_stride,
                         c.row_bytes, smem_u32(&full[st]), pol, c.hint);
            if (++st == c.nst) { st = 0; ph ^= 1; }
        }
        return;
    }
    if (warp < c.consumers) {
        int st = 0; uint32_t ph = 0;
        uint32_t acc = 0;
        for (long long i = 0; i < c.stages_per_cta; ++i) {
            mbar_wait(&full[st], ph);
            if (c.work) {
                const uint32_t a = ring + st * stage_bytes;
                const int per_warp = c.rows * c.row_bytes / c.consumers;     // bytes
                for (int k = lane * 16; k < per_warp; k += 512) {
                    const int off = warp * per_warp + k;
                    const int r = off / c.row_bytes, cc = off - r * c.row_bytes;
                    uint4 v;
                    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                                 : "r"(a + r * c.pitch + cc));
                    acc += v.x ^ v.y ^ v.z ^ v.w;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
            if (++st == c.nst) { st = 0; ph ^= 1; }
        }
        if (acc == 0x12345678u) out[0] = acc;
    }
}

int main() {
    const size_t bytes = (size_t)4 << 30;
    uint8_t* src; unsigned long long* out;
    cudaMalloc(&src, bytes); cudaMemset(src, 1, bytes); cudaMalloc(&out, 8);
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    struct V { const char* name; Cfg c; } vs[] = {
        {"16 x 2560 B, pitch 2624, 4 st, evict_first, work", {16, 2560, 2624, 4, 16, 1, 1, 5120, 0}},
        {"16 x 2560 B, pitch 2624, 4 st, evict_first, nowork", {16, 2560, 2624, 4, 16, 0, 1, 5120, 0}},
        {"16 x 2560 B, pitch 2624, 4 st, no hint, nowork", {16, 2560, 2624, 4, 16, 0, 0, 5120, 0}},
        {"16 x 2560 B, pitch 2560, 4 st, evict_first, nowork", {16, 2560, 2560, 4, 16, 0, 1, 5120, 0}},
        {"16 x 2560 B contiguous src, pitch 2560, 4 st", {16, 2560, 2560, 4, 16, 0, 1, 2560, 0}},
        {"8 x 5120 B, pitch 5184, 4 st", {8, 5120, 5184, 4, 16, 0, 1, 5120, 0}},
        {"1 x 40960 B, 4 st", {1, 40960, 40960, 4, 16, 0, 1, 40960, 0}},
        {"32 x 1280 B, pitch 1344, 4 st", {32, 1280, 1344, 4, 16, 0, 1, 5120, 0}},
        {"16 x 1280 B, pitch 1344, 8 st", {16, 1280, 1344, 8, 16, 0, 1, 5120, 0}},
        {"16 x 2560 B, pitch 2624, 2 st", {16, 2560, 2624, 2, 16, 0, 1, 5120, 0}},
        {"16 x 2560 B, pitch 2624, 3 st", {16, 2560, 2624, 3, 16, 0, 1, 5120, 0}},
        {"16 x 2560 B, pitch 2624, 5 st", {16, 2560, 2624, 5, 16, 0, 1, 5120, 0}},
    };
    for (auto& v : vs) {
        Cfg c = v.c;
        const size_t per_stage = (size_t)c.rows * c.row_bytes;
        c.stages_per_cta = (long long)(((size_t)3 << 30) / sms / ((size_t)c.rows * c.src_stride));
        const int stage_bytes = (c.rows * c.pitch + 127) / 128 * 128;
        const size_t smem = 1024 + (size_t)c.nst * stage_bytes;
        cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        stream_kernel<<<sms, 544, smem>>>(src, bytes, c, out);
        cudaEventRecord(e0);
        stream_kernel<<<sms, 544, smem>>>(src, bytes, c, out);
        cudaEventRecord(e1);
        cudaError_t err = cudaDeviceSynchronize();
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        const double gb = (double)per_stage * c.stages_per_cta * sms / 1e9;
        printf("%-55s %8.3f ms  %7.1f GB/s  (%s)\n", v.name, ms, gb / ms * 1e3, cudaGetErrorString(err));
    }
    return 0;
}
