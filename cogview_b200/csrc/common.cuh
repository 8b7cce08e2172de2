// Shared device-side primitives for the sm_90a kernels: mbarrier, TMA, wgmma and its shared-memory
// descriptors, warp reductions.  Everything is inline PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

namespace cv {

// ----------------------------------------------------------------------------------------------
// generic helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Programmatic dependent launch: let the next kernel in the stream start its prologue now / wait until the
// previous kernel has completed and its writes are visible.  Both are no-ops for a normally launched kernel.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// atomic max on a non-negative float stored as its bit pattern (monotone for x >= 0)
__device__ __forceinline__ void atomic_max_nonneg(float* addr, float v) {
    atomicMax(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// OpenAI tanh-GELU, reference mpu/sparse_transformer.py:172-176.  tanh(u) = 1 - 2/(exp(2u)+1).
__device__ __forceinline__ float gelu_tanh(float x) {
    float u = 0.7978845608028654f * x * (1.0f + 0.044715f * x * x);
    float t = 1.0f - 2.0f / (__expf(2.0f * u) + 1.0f);
    return 0.5f * x * (1.0f + t);
}
// Same function with the hardware tanh (MUFU.TANH, max relative error 2^-11 — below bf16's 2^-9 half-ulp), used
// where the result is rounded to bf16 anyway (GEMM epilogue): 6 instructions instead of ~30.
__device__ __forceinline__ float gelu_tanh_fast(float x) {
    float u = 0.7978845608028654f * x * (1.0f + 0.044715f * x * x);
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
    return 0.5f * x * (1.0f + t);
}
// d/dx of the above
__device__ __forceinline__ float gelu_tanh_grad(float x) {
    float x2 = x * x;
    float u = 0.7978845608028654f * x * (1.0f + 0.044715f * x2);
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
    float du = 0.7978845608028654f * (1.0f + 3.0f * 0.044715f * x2);
    return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * du;
}

// ----------------------------------------------------------------------------------------------
// Counter-based dropout (Philox4x32-10).  The keep-mask of element `idx` of dropout site `stream` is a pure
// function of (seed, stream, idx): the forward kernel that applies the mask and the backward kernel that needs it
// again regenerate it instead of storing it (torch.nn.Dropout of the reference: mpu/sparse_transformer.py:98,105,
// 224,425 — bitwise parity with torch's generator is neither possible nor needed; parity runs use p = 0).
// One call yields the random words of 4 consecutive elements (idx/4 is the counter).
// ----------------------------------------------------------------------------------------------
struct DropoutArgs {
    float p;             // drop probability; 0 disables
    float scale;         // 1 / (1 - p)
    uint32_t threshold;  // keep iff random word >= threshold (= p * 2^32)
    uint32_t stream;     // dropout site id
    uint64_t seed;
};
__device__ __forceinline__ uint4 philox4x32_10(uint64_t seed, uint64_t counter, uint32_t stream) {
    uint32_t c0 = (uint32_t)counter, c1 = (uint32_t)(counter >> 32), c2 = stream, c3 = 0x9E3779B9u;
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
}
// multiplies v[0..3] (elements idx4*4 .. idx4*4+3 of the site) by keep * scale
__device__ __forceinline__ void dropout4(const DropoutArgs& d, uint64_t idx4, float& a, float& b, float& c, float& e) {
    const uint4 r = philox4x32_10(d.seed, idx4, d.stream);
    a = r.x >= d.threshold ? a * d.scale : 0.f;
    b = r.y >= d.threshold ? b * d.scale : 0.f;
    c = r.z >= d.threshold ? c * d.scale : 0.f;
    e = r.w >= d.threshold ? e * d.scale : 0.f;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Spin on the phase parity.  A bounded wait (wall-clock, %globaltimer) turns a protocol bug into a trap
// (an error the host sees) instead of a hung GPU.
#ifndef CV_WAIT_TIMEOUT_NS
#define CV_WAIT_TIMEOUT_NS 4000000000ull
#endif
__device__ __forceinline__ uint64_t global_timer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// TRACE = false: no printf on the timeout path (a function call there would make ptxas serialise the wgmma of a
// warpgroup that waits with MMAs still in flight)
template <bool TRACE = true>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    uint32_t spins = 0;
    uint64_t t0 = 0;
    while (true) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) break;
        if ((++spins & 0x3ff) == 0) {
            const uint64_t now = global_timer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > CV_WAIT_TIMEOUT_NS) {
                if (TRACE)
                    printf("cogview_b200: mbarrier wait timed out (block %d,%d,%d thread %d, smem 0x%x, parity %u)\n",
                           blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x, addr, parity);
                __trap();
            }
        }
    }
}

// named barrier among a subset of warps (id 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
        : "memory");
}
// make generic-proxy smem writes visible to the async proxy (TMA store / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a): accumulators live in the registers of the 128 threads of a warpgroup
// ----------------------------------------------------------------------------------------------
// make the warpgroup's register / shared-memory writes visible to the wgmma that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the accumulator registers ordered around the asynchronous wgmma
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// move the register budget between the producer warpgroup and the MMA warpgroups
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// Accumulator fragment of an m64nN wgmma, thread t of the warpgroup (warp w = t / 32, lane l):
//   d[4i + e]     row 16w + l/4,      column 8i + 2(l%4) + e     (e = 0, 1)
//   d[4i + 2 + e] row 16w + l/4 + 8,  same column
// The A-from-registers fragment of a k16 slice uses the same positions: the bf16 pairs of d[8k .. 8k+7] of an
// accumulator are the A operand for k-columns 16k .. 16k+15 (frag_a below).
__device__ __forceinline__ void frag_a(const uint32_t* packed, int k, uint32_t (&a)[4]) {
    a[0] = packed[4 * k]; a[1] = packed[4 * k + 1]; a[2] = packed[4 * k + 2]; a[3] = packed[4 * k + 3];
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (PTX ISA "Matrix Descriptor Format"), 128-byte swizzle:
//   bits [0,14)  start address >> 4
//   bits [16,30) leading-dimension byte offset >> 4
//   bits [32,46) stride-dimension byte offset >> 4
//   bits [62,64) layout type: 1 = SWIZZLE_128B
// K-major operand (rows = M or N index, 128 bytes of K per row): 8-row groups SBO apart; LBO unused.
// MN-major operand (rows = K index, 128 bytes of M/N per row): 8-row K groups SBO apart, 64-element
// M/N chunks LBO apart.  Every tile here starts 1024-byte aligned, so the base-offset field stays 0; stepping
// along K inside a swizzled row is done by advancing the start address (32 bytes per k16 step, K-major).
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

}  // namespace cv

#include "wgmma.cuh"
