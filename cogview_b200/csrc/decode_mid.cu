// Decode kernels for 17..64 sequences per step (csrc/decode.cu covers 1..16 and is not touched by this file).
//
//   cv_linear_mid_m  : y[M,N] = x[M,K] W[N,K]^T + b (+GELU) (+abs-max), 17 <= M <= 64 — the contract of
//                      cv_linear_small_m (F.linear of mpu/layers.py:243,319 and the last-token logits GEMM,
//                      model/gpt2_modeling.py:117, as reached from the sampling loop, generation/sampling.py:147-151)
//   cv_ln_pair_mid_m : the Sandwich-LN glue of cv_ln_pair_small_m for 17 <= M <= 64 rows
//
// At 64 rows a linear still does only 64 FLOP per weight byte, far below the H100's ridge, so it stays a
// weight-streaming kernel; what changes against M <= 16 is that the activations no longer fit in MMA fragments
// held in registers, so the weights become the 64-row operand of a warpgroup MMA and the activations its N side.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;
typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------------
// thread-block cluster primitives
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_size() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
// every thread of every CTA of the cluster; shared-memory writes before it are visible cluster-wide after it
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// read a float at the same shared-memory offset in CTA `rank` of the cluster (distributed shared memory)
__device__ __forceinline__ float ld_dsmem_f32(uint32_t local_addr, uint32_t rank) {
    uint32_t remote;
    float v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_addr), "r"(rank));
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
    return v;
}

// ------------------------------------------------------------------------------------------------
// cv_linear_mid_m.
//
// Operands are swapped: D[128 weight rows x 64] += W_tile[128 x 64] . x_tile[64 x 64]^T, two consumer warpgroups
// (64 weight rows each, wgmma m64n64k16) sharing one x tile, so that x is read from L2 half as often as W from HBM.
// Rows M..63 of the x tile lie outside its tensor map and are zero-filled by the copy engine; they are never stored.
//
//   * grid = (S, ceil(N / 128)) in clusters of S CTAs: the S CTAs of a cluster own the same 128 weight rows and
//     split K between them, so that even N = 2560 (20 row tiles) gives every SM a stream;
//   * one producer thread issues the TMA loads (W with an L2 evict-first hint: it is read once per step) into a
//     ring of LM_STAGES x 24 KB, two CTAs per SM; weights do not depend on the previous kernel of the step, so
//     the first LM_STAGES weight tiles are requested BEFORE griddepcontrol.wait and only x after it;
//   * split-K reduction without global memory: every CTA leaves its fp32 partial tile in its own shared memory
//     (the drained ring), and after a cluster barrier rank r sums rows [128 r / S, 128 (r + 1) / S) of all S
//     partials through distributed shared memory in rank order 0..S-1 — a fixed order, so equal inputs give equal
//     bits on every replay — and applies bias / GELU / abs-max to them.
// ------------------------------------------------------------------------------------------------
constexpr int LM_BM = 128;                          // weight rows (output columns) per cluster
constexpr int LM_BK = 64;                           // 128 bytes of K per row: one swizzle row
constexpr int LM_MP = 64;                           // padded batch rows (wgmma N)
constexpr int LM_STAGES = 4;
constexpr int LM_W_BYTES = LM_BM * LM_BK * 2;
constexpr int LM_STAGE_BYTES = LM_W_BYTES + LM_MP * LM_BK * 2;
constexpr int LM_CONSUMERS = 256;                   // two warpgroups
constexpr int LM_THREADS = LM_CONSUMERS + 32;       // + the producer warp
constexpr int LM_PITCH = LM_BM + 4;                 // floats per batch row of the partial tile (conflict-free stores)
constexpr int LM_SMEM = 1024 + LM_STAGES * LM_STAGE_BYTES + 2 * LM_STAGES * 8;
static_assert(LM_MP * LM_PITCH * 4 <= LM_STAGES * LM_STAGE_BYTES, "the partial tile reuses the ring");

struct MidParams {
    const bf16* bias;
    void* out;
    int64_t ldo;
    int out_f32, act;
    float* absmax;
    int M, N, K;
};

__device__ __forceinline__ void tma_load_2d_evict_first(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                        uint64_t pol) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], "
        "[%2], %5;" ::"r"(smem_u32(smem)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(pol)
        : "memory");
}

__global__ void __launch_bounds__(LM_THREADS, 2)
linear_mid_m_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const MidParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + LM_STAGES * LM_STAGE_BYTES);
    uint64_t* empty_bar = full_bar + LM_STAGES;     // one arrive per consumer warp
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rank = cluster_rank(), S = cluster_size();
    const int n0 = blockIdx.y * LM_BM;
    const int kt_all = (p.K + LM_BK - 1) / LM_BK;
    const int kt0 = (int)(kt_all * rank / S), nk = (int)(kt_all * (rank + 1) / S) - kt0;   // this CTA's K tiles

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmW);
        tma_prefetch_desc(&tmX);
        for (int i = 0; i < LM_STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], LM_CONSUMERS / 32);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == LM_CONSUMERS / 32) {
        // ------------------------------ TMA producer ------------------------------
        if (lane == 0) {
            uint64_t pol;
            asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
            const int pre = min(nk, LM_STAGES);
            for (int it = 0; it < pre; ++it) {
                mbar_expect_tx(&full_bar[it], LM_STAGE_BYTES);
                tma_load_2d_evict_first(smem + it * LM_STAGE_BYTES, &tmW, &full_bar[it], (kt0 + it) * LM_BK, n0, pol);
            }
            // the weights are in flight: let the next kernel start its own prologue, then wait for the producer of x
            pdl_launch_dependents();
            pdl_wait();
            for (int it = 0; it < pre; ++it)
                tma_load_2d(smem + it * LM_STAGE_BYTES + LM_W_BYTES, &tmX, &full_bar[it], (kt0 + it) * LM_BK, 0);
            for (int it = pre; it < nk; ++it) {
                const int stage = it % LM_STAGES;
                mbar_wait<false>(&empty_bar[stage], (uint32_t)(it / LM_STAGES - 1) & 1u);
                uint8_t* dst = smem + stage * LM_STAGE_BYTES;
                mbar_expect_tx(&full_bar[stage], LM_STAGE_BYTES);
                tma_load_2d_evict_first(dst, &tmW, &full_bar[stage], (kt0 + it) * LM_BK, n0, pol);
                tma_load_2d(dst + LM_W_BYTES, &tmX, &full_bar[stage], (kt0 + it) * LM_BK, 0);
            }
        } else {
            pdl_launch_dependents();
        }
    } else {
        // ------------------------------ wgmma consumers ------------------------------
        pdl_launch_dependents();
        const int wg = warp >> 2;                   // weight rows 64 wg .. 64 wg + 63 of the tile
        float acc[LM_MP / 2];
#pragma unroll
        for (int i = 0; i < LM_MP / 2; ++i) acc[i] = 0.f;
        for (int it = 0; it < nk; ++it) {
            const int stage = it % LM_STAGES;
            mbar_wait<false>(&full_bar[stage], (uint32_t)(it / LM_STAGES) & 1u);
            const uint32_t a_addr = smem_u32(smem + stage * LM_STAGE_BYTES) + wg * (64 * 128);
            const uint32_t b_addr = smem_u32(smem + stage * LM_STAGE_BYTES + LM_W_BYTES);
            fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < LM_BK / 16; ++k)
                wgmma_ss_n64<0, 0>(acc, make_smem_desc_sw128(a_addr + k * 32, 0, 1024),
                                   make_smem_desc_sw128(b_addr + k * 32, 0, 1024), (it | k) != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();                        // a 24 KB stage takes far longer to arrive than to multiply
            fence_regs(acc);
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
        }
        // both warpgroups are done with the ring: it now holds this CTA's partial tile, part[batch row][weight row]
        named_bar_sync(1, LM_CONSUMERS);
        float* part = reinterpret_cast<float*>(smem);
        const int r_in = 64 * wg + 16 * (warp & 3) + (lane >> 2), c_in = 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < LM_MP / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                part[(8 * i + c_in + e) * LM_PITCH + r_in] = acc[4 * i + e];
                part[(8 * i + c_in + e) * LM_PITCH + r_in + 8] = acc[4 * i + 2 + e];
            }
        }
    }
    __syncwarp();                                   // the producer lane rejoins its warp: the barrier is warp-aligned
    cluster_sync();
    if (warp < LM_CONSUMERS / 32) {
        pdl_wait();                                 // `out` / `absmax` may still be in use by earlier kernels
        const int width = LM_BM / (int)S, n_lo = (int)rank * width;
        const uint32_t part_addr = smem_u32(smem);
        float tmax = 0.f;
        for (int idx = threadIdx.x; idx < p.M * width; idx += LM_CONSUMERS) {
            const int nn = n_lo + idx % width, m = idx / width;    // consecutive threads -> consecutive columns
            const int n = n0 + nn;
            if (n >= p.N) continue;
            float v = 0.f;
            for (uint32_t r = 0; r < S; ++r) v += ld_dsmem_f32(part_addr + (uint32_t)(m * LM_PITCH + nn) * 4u, r);
            if (p.bias != nullptr) v += __bfloat162float(p.bias[n]);
            if (p.act == 1) v = gelu_tanh(v);
            if (p.out_f32) {
                static_cast<float*>(p.out)[(size_t)m * p.ldo + n] = v;
                tmax = fmaxf(tmax, fabsf(v));
            } else {
                const bf16 o = __float2bfloat16_rn(v);
                static_cast<bf16*>(p.out)[(size_t)m * p.ldo + n] = o;
                tmax = fmaxf(tmax, fabsf(__bfloat162float(o)));
            }
        }
        if (p.absmax != nullptr) {
            tmax = warp_max(tmax);
            if (lane == 0 && tmax > 0.f) atomic_max_nonneg(p.absmax, tmax);
        }
    }
    cluster_sync();                                 // no CTA leaves while its partial tile is being read
}

// ------------------------------------------------------------------------------------------------
// cv_ln_pair_mid_m: one cluster of ceil(M / 8) CTAs, 8 rows per CTA, 4 warps per row.
//   y  = res_in + LN_post(gemm_out / (max|gemm_out| / 8))
//   xn = LN_pre(y / (max|y| / 8))
// (mpu/sparse_transformer.py:326-331 and :337-340 + :319 of the next layer.)  max|y| is over ALL rows: every CTA
// publishes the maximum of its rows in its shared memory and reads the others' through distributed shared memory
// after one cluster barrier.  Per row the arithmetic — and the order of every row reduction — is that of the 8-row
// instance of ln_pair_kernel (csrc/decode.cu), so y is bit-equal to what cv_ln_pair_small_m gives for the same rows.
// ------------------------------------------------------------------------------------------------
constexpr int LP_THREADS = 1024;
constexpr int LP_ROWS = 8;                          // rows per CTA
constexpr int LP_WPR = 32 / LP_ROWS;                // warps per row
constexpr int LP_TPR = LP_WPR * 32;                 // threads per row

// NP: bf16 pairs per thread (K <= 2 * NP * LP_TPR)
template <int NP>
__global__ void __launch_bounds__(LP_THREADS)
ln_pair_mid_kernel(const float* __restrict__ res_in, const bf16* __restrict__ gemm_out,
                   const float* __restrict__ absmax_gemm, const bf16* __restrict__ g_post,
                   const bf16* __restrict__ b_post, const bf16* __restrict__ g_pre, const bf16* __restrict__ b_pre,
                   float eps, float* __restrict__ res_out, bf16* __restrict__ xn_out, int M, int K) {
    __shared__ float red[4][LP_ROWS][LP_WPR];
    __shared__ float smax[32];
    __shared__ float cta_max;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slot = warp / LP_WPR, wr = warp % LP_WPR;
    const int row = (int)cluster_rank() * LP_ROWS + slot;
    const int tr = wr * 32 + lane;                  // thread index within the row group
    const bool row_ok = row < M;
    const bool has_post = gemm_out != nullptr;

    pdl_launch_dependents();
    pdl_wait();

    auto row_reduce = [&](float s, int buf) -> float {   // sum over the row group; one barrier per call
        s = warp_sum(s);
        if (lane == 0) red[buf][slot][wr] = s;
        __syncthreads();
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < LP_WPR; ++i) t += red[buf][slot][i];
        return t;
    };
    // LayerNorm parameters (packed bf16x2) and the residual are read where they are used: with 1024 threads a thread
    // has 64 registers, not enough to hold them next to the row
    auto param = [&](const bf16* q, int e) -> uint32_t {
        const int k = 2 * (tr + e * LP_TPR);
        return k < K ? __ldg(reinterpret_cast<const uint32_t*>(q + k)) : 0u;
    };
    auto lo = [](uint32_t u) { return __uint_as_float(u << 16); };
    auto hi = [](uint32_t u) { return __uint_as_float(u & 0xffff0000u); };

    float2 v[NP];
    const float inv_k = 1.0f / K;
    if (has_post) {
        uint32_t go[NP];
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            const int k = 2 * (tr + e * LP_TPR);
            go[e] = (k < K && row_ok) ? *reinterpret_cast<const uint32_t*>(gemm_out + (size_t)row * K + k) : 0u;
        }
        const float c = *absmax_gemm * 0.125f;
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < NP; ++e) { v[e] = make_float2(lo(go[e]), hi(go[e])); s += v[e].x + v[e].y; }
        const float mean = row_reduce(s, 0) * inv_k;
        float ss = 0.f;
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            if (2 * (tr + e * LP_TPR) < K) {
                const float a = v[e].x - mean, b = v[e].y - mean;
                ss += a * a + b * b;
            }
        }
        const float var = row_reduce(ss, 1) * inv_k;
        const float rstd = rsqrtf(var + eps * c * c);
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            const int k = 2 * (tr + e * LP_TPR);
            const float2 rs = (k < K && row_ok) ? *reinterpret_cast<const float2*>(res_in + (size_t)row * K + k)
                                                : make_float2(0.f, 0.f);
            const uint32_t gp = param(g_post, e), bp = param(b_post, e);
            v[e].x = (v[e].x - mean) * rstd * lo(gp) + lo(bp) + rs.x;
            v[e].y = (v[e].y - mean) * rstd * hi(gp) + hi(bp) + rs.y;
        }
    } else {
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            const int k = 2 * (tr + e * LP_TPR);
            v[e] = (k < K && row_ok) ? *reinterpret_cast<const float2*>(res_in + (size_t)row * K + k)
                                     : make_float2(0.f, 0.f);
        }
    }
    float mx = 0.f, s = 0.f;
#pragma unroll
    for (int e = 0; e < NP; ++e) {
        const int k = 2 * (tr + e * LP_TPR);
        if (k < K && row_ok) {
            if (res_out != nullptr) *reinterpret_cast<float2*>(res_out + (size_t)row * K + k) = v[e];
            mx = fmaxf(mx, fmaxf(fabsf(v[e].x), fabsf(v[e].y)));
            s += v[e].x + v[e].y;
        }
    }
    mx = warp_max(mx);
    s = warp_sum(s);
    if (lane == 0) { smax[warp] = mx; red[2][slot][wr] = s; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) m = fmaxf(m, smax[i]);
        cta_max = m;
    }
    cluster_sync();
    float am = 0.f;
    const uint32_t ranks = cluster_size(), max_addr = smem_u32(&cta_max);
    for (uint32_t r = 0; r < ranks; ++r) am = fmaxf(am, ld_dsmem_f32(max_addr, r));
    float tsum = 0.f;
#pragma unroll
    for (int i = 0; i < LP_WPR; ++i) tsum += red[2][slot][i];
    const float mean = tsum * inv_k;
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < NP; ++e) {
        if (2 * (tr + e * LP_TPR) < K && row_ok) {
            const float a = v[e].x - mean, b = v[e].y - mean;
            ss += a * a + b * b;
        }
    }
    const float var = row_reduce(ss, 3) * inv_k;
    const float c = am * 0.125f;
    const float rstd = rsqrtf(var + eps * c * c);
#pragma unroll
    for (int e = 0; e < NP; ++e) {
        const int k = 2 * (tr + e * LP_TPR);
        if (k < K && row_ok) {
            const uint32_t gq = param(g_pre, e), bq = param(b_pre, e);
            const float a = (v[e].x - mean) * rstd * lo(gq) + lo(bq);
            const float b = (v[e].y - mean) * rstd * hi(gq) + hi(bq);
            *reinterpret_cast<uint32_t*>(xn_out + (size_t)row * K + k) = pack_bf16x2(a, b);
        }
    }
    cluster_sync();                                 // no CTA leaves while its maximum is being read
}

// one cluster spanning grid.x (the K split of a row tile, or the row groups of the LayerNorm pair), launched with
// programmatic dependent launch allowed
template <typename... KArgs, typename... Args>
cudaError_t launch_cluster_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                               Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = grid.x;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = cvh::pdl_enabled() ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace

extern "C" int cv_linear_mid_m(const void* x, int64_t ldx, const void* W, int64_t ldw, const void* bias, void* out,
                               int64_t ldo, int out_is_f32, int act, float* absmax, int M, int N, int K, void* stream) {
    CV_REQUIRE(x && W && out, "null pointer");
    CV_REQUIRE(M >= 17 && M <= 64, "cv_linear_mid_m handles 17 <= M <= 64 rows (cv_linear_small_m below, cv_gemm_bf16 above)");
    CV_REQUIRE(N > 0 && K > 0 && K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "K, ldx, ldw must be multiples of 8");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
               "x and W must be 16-byte aligned");
    CV_REQUIRE(act == 0 || act == 1, "act must be 0 or 1");
    const int tiles = (N + LM_BM - 1) / LM_BM, kt = (K + LM_BK - 1) / LM_BK;
    CV_REQUIRE(tiles <= 65535, "N too large");
    // split K (cluster size 1, 2, 4 or 8) until every SM has a CTA, as long as a CTA keeps >= 4 K tiles to pipeline
    int S = 1;
    while (S < 8 && tiles * S < cvh::num_sms() && kt / (2 * S) >= 4) S *= 2;
    alignas(64) CUtensorMap tmW, tmX;
    int rc = cvh::encode_tmap_2d_bf16(&tmW, W, N, K, ldw, LM_BM, LM_BK);
    if (rc) return rc;
    rc = cvh::encode_tmap_2d_bf16(&tmX, x, M, K, ldx, LM_MP, LM_BK);      // rows M..63 of a box: zero fill
    if (rc) return rc;
    MidParams p;
    p.bias = static_cast<const bf16*>(bias);
    p.out = out; p.ldo = ldo; p.out_f32 = out_is_f32; p.act = act; p.absmax = absmax;
    p.M = M; p.N = N; p.K = K;
    CV_CUDA(cudaFuncSetAttribute(linear_mid_m_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LM_SMEM));
    CV_CUDA(launch_cluster_pdl(linear_mid_m_kernel, dim3(S, tiles), dim3(LM_THREADS), LM_SMEM,
                               static_cast<cudaStream_t>(stream), tmW, tmX, p));
    cvh::count_launches(1);
    return 0;
}

extern "C" int cv_ln_pair_mid_m(const float* res_in, const void* gemm_out, const float* absmax_gemm, const void* g_post,
                                const void* b_post, const void* g_pre, const void* b_pre, float eps, float* res_out,
                                void* xn_out, int M, int K, void* stream) {
    CV_REQUIRE(res_in && g_pre && b_pre && xn_out, "null pointer");
    CV_REQUIRE(gemm_out == nullptr || (absmax_gemm && g_post && b_post), "gemm_out needs absmax_gemm, g_post, b_post");
    CV_REQUIRE(M >= 17 && M <= 64 && K > 0 && K % 2 == 0, "17 <= M <= 64, K even");
    const int need = (K + 2 * LP_TPR - 1) / (2 * LP_TPR);      // bf16 pairs per thread
    CV_REQUIRE(need <= 10, "K too large for cv_ln_pair_mid_m (K <= 2560)");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bf16* go = static_cast<const bf16*>(gemm_out);
    const bf16 *gp = static_cast<const bf16*>(g_post), *bp = static_cast<const bf16*>(b_post);
    const bf16 *gq = static_cast<const bf16*>(g_pre), *bq = static_cast<const bf16*>(b_pre);
    bf16* xo = static_cast<bf16*>(xn_out);
    const dim3 grid((M + LP_ROWS - 1) / LP_ROWS);
#define LP(NP_)                                                                                                       \
    CV_CUDA(launch_cluster_pdl(ln_pair_mid_kernel<NP_>, grid, dim3(LP_THREADS), 0, s, res_in, go, absmax_gemm, gp, bp, \
                               gq, bq, eps, res_out, xo, M, K))
    if (need <= 2) LP(2);
    else if (need <= 5) LP(5);
    else LP(10);
#undef LP
    cvh::count_launches(1);
    return 0;
}
