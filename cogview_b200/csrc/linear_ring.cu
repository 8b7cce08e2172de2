// Weight-streaming linear for the decode step (M <= 8 rows): y[M,N] = x[M,K] W[N,K]^T + bias (+GELU) (+abs-max).
//
// Reference: F.linear of mpu/layers.py:243,319 and the last-token logits GEMM (model/gpt2_modeling.py:117) as reached
// from the sampling loop (generation/sampling.py:147-151).  Same contract as linear_small_m_kernel (csrc/decode.cu);
// cv_linear_small_m picks this kernel when the shape allows it.
//
// Why a second kernel: the fragment-direct loads of linear_small_m_kernel read HBM in 64-byte pieces through the LSU;
// bulk copies of whole row segments into a shared-memory ring keep more bytes in flight per SM.  The machinery is the
// one the persistent step kernel (csrc/decode_step.cu) is built on:
//   * 2 CTAs per SM, each owning a contiguous row range of W; per CTA 8 consumer warps + 1 producer warp + 1
//     epilogue warp, ~100 KB of shared memory — small enough for the NEXT linear of the step to become resident
//     (programmatic dependent launch) and start streaming ITS weights while this one finishes: weights never depend
//     on the previous kernel, only x does (griddepcontrol.wait sits in front of the first read of x / first store);
//   * producer: cp.async.bulk of 16-row x 512-column slabs (one bulk copy per row segment, L2 evict-first) into a
//     byte ring, mbarrier per stage;
//   * consumers: K slices of a stage, mma.sync.m16n8k16 with the weights as A (16 output columns as rows) and the
//     activations as B (sequences as columns), fragments by conflict-free 16-byte shared loads (row pitch = 64 mod
//     128 B), B fragments of a K chunk held in registers for all row tiles;
//   * K > 2560: chunks of 2560 columns, the activations of chunk k+1 copied (cp.async) while chunk k is multiplied,
//     the accumulators of the CTA's <= 2 row tiles carried across chunks;
//   * epilogue warp: sums the 8 K-slice partials of a finished tile, bias / GELU / abs-max, stores — the consumers
//     only bar.arrive.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;
typedef __nv_bfloat16 bf16;

constexpr int LW = 8;               // consumer warps = K slices of a stage
constexpr int LT = LW * 32;
constexpr int LCE = LT + 32;        // consumers + epilogue warp
constexpr int LNT = LT + 64;        // + producer warp + epilogue warp
constexpr int TILE = 16;
constexpr int NB = 16;              // mbarrier pairs of the byte ring
constexpr int KCHUNK = 2560;        // K columns per operand chunk
enum { BAR_CONS = 1, BAR_PFULL = 2, BAR_PFREE = 4 };

struct LParams {
    const bf16* x; int64_t ldx;
    const bf16* W; int64_t ldw;
    const bf16* bias;
    void* out; int64_t ldo;
    int out_f32, act;
    float* absmax;
    int M, N, K;
    int kchunk, nq, kstage, pitch, xpitch, xbuf_bytes, ring_bytes;
};

constexpr int SM_BAR = 0;                                  // full[NB], empty[NB]
constexpr int SM_ASZ = 2 * NB * 8;                         // uint32 asz[NB]
constexpr int SM_PART = 512;                               // float part[2][LW][TILE][8]
constexpr int SM_XOP = SM_PART + 2 * LW * TILE * 8 * 4;    // 8704: multiple of 128

__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
    return r;
}
__device__ __forceinline__ void sts128(uint32_t a, const uint4& v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol)
        : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ uint64_t evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                          uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t mbar_try(uint32_t addr, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    return done;
}
__device__ __noinline__ void ring_wait_slow(uint32_t addr, uint32_t parity) {
    uint32_t spins = 0;
    uint64_t t0 = 0;
    while (!mbar_try(addr, parity)) {
        if ((++spins & 0x3ff) == 0) {
            const uint64_t now = global_timer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > CV_WAIT_TIMEOUT_NS) {
                printf("cogview_b200: linear_ring_kernel wait timed out (block %d, thread %d)\n", blockIdx.x, threadIdx.x);
                __trap();
            }
        }
    }
}
__device__ __forceinline__ void ring_wait(uint32_t addr, uint32_t parity) {
    if (!mbar_try(addr, parity)) ring_wait_slow(addr, parity);
}

template <int MR, int CPW, int NKS>
__global__ void __launch_bounds__(LNT, MR == 4 ? 2 : 1) linear_ring_kernel(const __grid_constant__ LParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + SM_BAR);
    uint64_t* empty = full + NB;
    float* part = reinterpret_cast<float*>(smem + SM_PART);
    const uint32_t xop = smem_u32(smem + SM_XOP);
    const uint32_t ring = xop + 2 * p.xbuf_bytes;
    const uint32_t full0 = smem_u32(full), empty0 = smem_u32(empty);
    const uint32_t R = (uint32_t)p.ring_bytes;
    const int M = p.M;
    // contiguous, byte-balanced row range of this CTA (N gridDim < 2^32)
    const int r0 = (int)(((unsigned int)p.N * blockIdx.x) / gridDim.x);
    const int r1 = (int)(((unsigned int)p.N * (blockIdx.x + 1u)) / gridDim.x);

    if (tid == 0) {
        for (int i = 0; i < NB; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], LW);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();          // the next kernel of the step may become resident and start ITS weight stream

    // ---- producer warp: weights do not depend on the previous kernel -> no griddepcontrol.wait here ----
    if (warp == LW) {
        const uint64_t pol = evict_first_policy();
        volatile uint32_t* asz = reinterpret_cast<volatile uint32_t*>(smem + SM_ASZ);
        int si = 0, tail = 0;
        uint32_t off = 0, used = 0;
#pragma unroll 1
        for (int kq = 0; kq < p.nq; ++kq) {
#pragma unroll 1
            for (int r = r0; r < r1; r += TILE) {
                const int rows = min(TILE, r1 - r);
                const bf16* src = p.W + (size_t)(r + min(lane, rows - 1)) * p.ldw + (size_t)kq * p.kchunk;
                const uint32_t size = (uint32_t)(rows * p.pitch + 127) & ~127u;
#pragma unroll 1
                for (int ks = 0; ks < NKS; ++ks) {
                    const bool wrap = off + size > R;       // a stage never wraps: skip the end of the ring
                    const uint32_t need = size + (wrap ? R - off : 0u);
                    while (used + need > R || tail + NB <= si) {
                        ring_wait(empty0 + (tail & (NB - 1)) * 8, (uint32_t)(tail / NB) & 1u);
                        used -= asz[tail & (NB - 1)];
                        ++tail;
                    }
                    if (wrap) off = 0;
                    const int b = si & (NB - 1);
                    asz[b] = need;
                    const uint32_t dst = ring + off;
                    off += size;
                    used += need;
                    if (lane == 0) mbar_expect_tx(&full[b], (uint32_t)(rows * p.kstage * 2));
                    __syncwarp();
                    if (lane < rows)
                        bulk_g2s(dst + lane * p.pitch, src + ks * p.kstage, (uint32_t)(p.kstage * 2), full0 + b * 8, pol);
                    ++si;
                }
            }
        }
        return;
    }

    // ---- epilogue warp ----
    if (warp == LW + 1) {
        named_bar_arrive(BAR_PFREE + 0, LCE);
        named_bar_arrive(BAR_PFREE + 1, LCE);
        const int nn = lane >> 1, mi0 = (lane & 1) * 4;
        int pbuf = 0;
        float tmax = 0.f;
        pdl_wait();                    // `out` / `absmax` may still be in use by the previous kernels of the stream
#pragma unroll 1
        for (int r = r0; r < r1; r += TILE) {
            const int n = r + nn;
            float bias_v = 0.f;
            if (p.bias != nullptr) bias_v = __bfloat162float(p.bias[min(n, r1 - 1)]);
            named_bar_sync(BAR_PFULL + pbuf, LCE);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int w = 0; w < LW; ++w) {
                const float4 x = *reinterpret_cast<const float4*>(part + ((pbuf * LW + w) * TILE + nn) * 8 + mi0);
                v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
            }
            named_bar_arrive(BAR_PFREE + pbuf, LCE);
            pbuf ^= 1;
            if (n < r1) {
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int mi = mi0 + j;
                    if (mi < M) {
                        float y = vv[j] + bias_v;
                        if (p.act == 1) y = gelu_tanh(y);
                        if (p.out_f32) {
                            static_cast<float*>(p.out)[(size_t)mi * p.ldo + n] = y;
                            tmax = fmaxf(tmax, fabsf(y));
                        } else {
                            const bf16 o = __float2bfloat16_rn(y);
                            static_cast<bf16*>(p.out)[(size_t)mi * p.ldo + n] = o;
                            tmax = fmaxf(tmax, fabsf(__bfloat162float(o)));
                        }
                    }
                }
            }
        }
        if (p.absmax != nullptr) {
            tmax = warp_max(tmax);
            if (lane == 0 && tmax > 0.f) atomic_max_nonneg(p.absmax, tmax);
        }
        return;
    }

    // ---- consumer warps ----
    const int g = lane >> 2, q = lane & 3;
    const int kpw = p.kstage / LW;                 // k elements per warp and stage ( = 32 * CPW )
    int pbuf = 0, sq = 0;
    uint32_t roff = 0;
    // rows >= M of the operand buffers stay zero
    for (int i = tid; i < 2 * p.xbuf_bytes / 16; i += LT) sts128(xop + i * 16, make_uint4(0, 0, 0, 0));
    named_bar_sync(BAR_CONS, LT);
    pdl_wait();                                    // x is written by the previous kernel
    auto xcopy = [&](const bf16* src, uint32_t dst) {
        const int vpr = p.kchunk >> 3;
#pragma unroll 1
        for (int mi = 0; mi < M; ++mi)
            for (int c = tid; c < vpr; c += LT) cp_async16(dst + mi * p.xpitch + c * 16, src + (size_t)mi * p.ldx + c * 8);
    };
    xcopy(p.x, xop);
    const bool two_tiles = p.nq > 1 && r1 - r0 > TILE;
    float dA[4] = {0.f, 0.f, 0.f, 0.f}, dB[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int kq = 0; kq < p.nq; ++kq) {
        cp_async_wait_all();                       // chunk kq has landed; every warp is done with chunk kq - 1
        named_bar_sync(BAR_CONS, LT);
        const uint32_t xb = xop + (kq & 1) * p.xbuf_bytes;
        if (kq + 1 < p.nq) xcopy(p.x + (size_t)(kq + 1) * p.kchunk, xop + ((kq + 1) & 1) * p.xbuf_bytes);
        const bool last = kq == p.nq - 1;
        uint4 xv[NKS][CPW];                        // B fragments of this chunk: read once, used by every row tile
#pragma unroll
        for (int ks = 0; ks < NKS; ++ks)
#pragma unroll
            for (int c = 0; c < CPW; ++c)
                xv[ks][c] = (MR == 8 || g < MR)
                                ? lds128(xb + g * p.xpitch + (ks * p.kstage + warp * kpw + q * 8) * 2 + c * 64)
                                : make_uint4(0, 0, 0, 0);
#pragma unroll 1
        for (int r = r0; r < r1; r += TILE) {
            const int rows = min(TILE, r1 - r);    // rows past the range are not in the stage: re-read the last one
            const uint32_t size = (uint32_t)(rows * p.pitch + 127) & ~127u;
            const uint32_t ra = min(g, rows - 1) * p.pitch + (warp * kpw + q * 8) * 2;
            const uint32_t rb = min(g + 8, rows - 1) * p.pitch + (warp * kpw + q * 8) * 2;
#pragma unroll
            for (int ks = 0; ks < NKS; ++ks) {
                if (roff + size > R) roff = 0;
                const uint32_t sa = ring + roff;
                roff += size;
                const int b = sq & (NB - 1);
                ring_wait(full0 + b * 8, (uint32_t)(sq / NB) & 1u);
                uint4 w0[CPW], w1[CPW];
#pragma unroll
                for (int c = 0; c < CPW; ++c) {
                    w0[c] = lds128(sa + ra + c * 64);
                    w1[c] = lds128(sa + rb + c * 64);
                }
#pragma unroll
                for (int c = 0; c < CPW; ++c) {
                    mma_16816(dA, w0[c].x, w1[c].x, w0[c].y, w1[c].y, xv[ks][c].x, xv[ks][c].y);
                    mma_16816(dA, w0[c].z, w1[c].z, w0[c].w, w1[c].w, xv[ks][c].z, xv[ks][c].w);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[b]);
                ++sq;
            }
            if (last) {
                // D fragment: d0,d1 = (row g, cols 2q,2q+1), d2,d3 = (row g+8, ...); row = output column, col = sequence
                named_bar_sync(BAR_PFREE + pbuf, LCE);       // the epilogue warp has read this buffer (two tiles ago)
                float* pw = part + ((pbuf * LW + warp) * TILE) * 8;
                pw[g * 8 + 2 * q] = dA[0];
                pw[g * 8 + 2 * q + 1] = dA[1];
                pw[(g + 8) * 8 + 2 * q] = dA[2];
                pw[(g + 8) * 8 + 2 * q + 1] = dA[3];
                dA[0] = dA[1] = dA[2] = dA[3] = 0.f;
                named_bar_arrive(BAR_PFULL + pbuf, LCE);
                pbuf ^= 1;
            }
            if (two_tiles) {
#pragma unroll
                for (int i = 0; i < 4; ++i) { const float tmp = dA[i]; dA[i] = dB[i]; dB[i] = tmp; }
            }
        }
    }
}

}  // namespace

namespace cvh {

// Returns 1 if the shape is not handled here (the caller falls back to linear_small_m_kernel), 0 on launch,
// or an error code.
int linear_ring(const void* x, int64_t ldx, const void* W, int64_t ldw, const void* bias, void* out, int64_t ldo,
                int out_is_f32, int act, float* absmax, int M, int N, int K, cudaStream_t s) {
    if (M < 1 || M > 8 || K % 256 != 0 || (K > KCHUNK && K % KCHUNK != 0)) return 1;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(W) & 15) || ldx % 8 || ldw % 8) return 1;
    LParams p;
    p.x = static_cast<const bf16*>(x); p.ldx = ldx;
    p.W = static_cast<const bf16*>(W); p.ldw = ldw;
    p.bias = static_cast<const bf16*>(bias);
    p.out = out; p.ldo = ldo; p.out_f32 = out_is_f32; p.act = act; p.absmax = absmax;
    p.M = M; p.N = N; p.K = K;
    p.kchunk = K > KCHUNK ? KCHUNK : K;
    p.nq = K / p.kchunk;
    int kstage = 256;
    for (int k = 256; k <= 768; k += 256)
        if (p.kchunk % k == 0) kstage = k;
    p.kstage = kstage;
    const int nks = p.kchunk / kstage, cpw = kstage / 256;
    p.pitch = kstage * 2 + 64;
    p.xpitch = p.kchunk * 2 + 64;
    const int MR = M <= 4 ? 4 : 8;
    p.xbuf_bytes = (MR * p.xpitch + 127) / 128 * 128;
    const int per_sm = MR == 4 ? 2 : 1;
    int grid = per_sm * num_sms();
    if (grid > N) grid = N;
    if (p.nq > 1 && (N + grid - 1) / grid > 2 * TILE) return 1;      // accumulators of <= 2 row tiles are carried
    if ((int64_t)N * (grid + 1) >= (1ll << 32)) return 1;
    const int stage = (TILE * p.pitch + 127) / 128 * 128;
    int max_smem = 0, dev = 0;
    CV_CUDA(cudaGetDevice(&dev));
    CV_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const int fixed = SM_XOP + 2 * p.xbuf_bytes;
    // 2 CTAs per SM (M <= 4): ~100 KB each; otherwise whatever one CTA can get
    int budget = per_sm == 2 ? (max_smem + 1024) / 2 - 2048 : max_smem - 1024;
    int ring_bytes = (budget - fixed) / 128 * 128;
    if (ring_bytes < 2 * stage) {
        ring_bytes = 2 * stage;
        if (fixed + ring_bytes > max_smem) return 1;
    }
    p.ring_bytes = ring_bytes;
    const size_t smem_bytes = (size_t)fixed + (size_t)ring_bytes;

    typedef void (*KernelFn)(const LParams);
    KernelFn fn = nullptr;
#define LR_PICK(MR_)                                                                 \
    if (cpw == 2 && nks == 5) fn = linear_ring_kernel<MR_, 2, 5>;                    \
    else if (cpw == 2 && nks == 2) fn = linear_ring_kernel<MR_, 2, 2>;               \
    else if (cpw == 2 && nks == 1) fn = linear_ring_kernel<MR_, 2, 1>;               \
    else if (cpw == 3 && nks == 1) fn = linear_ring_kernel<MR_, 3, 1>;               \
    else if (cpw == 1 && nks == 1) fn = linear_ring_kernel<MR_, 1, 1>;               \
    else if (cpw == 3 && nks == 2) fn = linear_ring_kernel<MR_, 3, 2>;               \
    else if (cpw == 2 && nks == 4) fn = linear_ring_kernel<MR_, 2, 4>;               \
    else if (cpw == 2 && nks == 3) fn = linear_ring_kernel<MR_, 2, 3>;
    if (MR == 4) { LR_PICK(4) } else { LR_PICK(8) }
#undef LR_PICK
    if (fn == nullptr) return 1;
    CV_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    CV_CUDA(launch_pdl(fn, dim3(grid), dim3(LNT), smem_bytes, s, true, p));
    count_launches(1);
    return 0;
}

}  // namespace cvh
