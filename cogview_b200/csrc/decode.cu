// Autoregressive-decode kernels (one new token per sequence per step).  At batch <= 16 every linear layer
// is a weight-streaming problem: the 7.86 GB of bf16 weights are read once per step and HBM bandwidth is
// the bound (SURVEY §8(d)), so these are coalesced CUDA-core kernels, not tensor-core tiles.
//
//   cv_linear_small_m : y[M,N] = x[M,K] W[N,K]^T + b (+GELU) (+abs-max), M <= 16
//                       (F.linear of mpu/layers.py:243,319 as reached from the sampling loop,
//                        generation/sampling.py:147-151, and the last-token logits GEMM, model/gpt2_modeling.py:117)
//   cv_attn_decode    : one query per sequence against the K|V cache, with the new token's K/V appended
//                       in the same kernel (standard_attention, mpu/sparse_transformer.py:652-673, for sq = 1,
//                       where every cached key is visible); with row_pad, a cache length per sequence
//                       (t_b = cur_len - row_pad[b]), so captions of different lengths share one decode batch
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

// ------------------------------------------------------------------------------------------------
// skinny linear on warp-level tensor-core MMAs (mma.sync m16n8k16, bf16 x bf16 -> fp32).
//
// 2 CTAs per SM each own a contiguous, byte-balanced range of output columns (rows of W) walked in MMA tiles of 16;
// the CTA's 8 warps split K, so even a 2560-column layer keeps 16 warps per SM streaming.  Per 32-element K chunk a lane issues two 16-byte loads of W (rows g and g+8,
// elements 8q..8q+7; g = lane/4, q = lane%4) and one 16-byte load of x (row g): because a dot product does not
// care in which order k is summed, those 8 contiguous elements are fed to two MMAs as the fragment slots
// {2q,2q+1,2q+8,2q+9}, with x permuted identically — so both operands are read with full 16-byte, sector-exact
// loads straight from global/L2 into MMA fragments (no shared memory, no conversions, ~10 instructions per KB of
// weights).  Four chunks (4 KB of W per warp) are in flight while the previous four are consumed.
// Partial [16 x 8] tiles of the 8 warps are reduced through shared memory; bias / GELU / abs-max in the epilogue.
// ------------------------------------------------------------------------------------------------
constexpr int SK_WARPS = 8;
constexpr int SK_NT = 16;         // output columns per CTA
constexpr int SK_UNROLL = 8;      // K chunks (of 32) in flight per warp: 512 contiguous bytes of each of its 16 rows

__device__ __forceinline__ void bf16x8_to_float(const uint4& u, float (&f)[8]) {
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        f[2 * t] = __low2float(p[t]);
        f[2 * t + 1] = __high2float(p[t]);
    }
}
// weights are read once per step: bypass L1 and mark the L2 lines evict-first so that the small hot tensors
// (activations, LayerNorm parameters, abs-max scalars) stay L2-resident while 7.9 GB of weights stream through
__device__ __forceinline__ uint64_t make_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint4 ld_stream(const void* p, uint64_t pol) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// WIDE: 9..16 rows of x — a second B fragment set (rows 8..15) and a second accumulator reuse the same weight
// fragments, so the weights are still streamed ONCE (two passes of the 8-row kernel would stream them twice); half the
// K chunks in flight per warp keeps the register count.
template <int UNROLL, bool WIDE>
struct SkStage {
    uint4 w0[UNROLL], w1[UNROLL], xv[UNROLL], xw[WIDE ? UNROLL : 1];
};

template <int UNROLL, bool WIDE>
__global__ void __launch_bounds__(SK_WARPS * 32, 2)
linear_small_m_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ W,
                      int64_t ldw, const __nv_bfloat16* __restrict__ bias, void* __restrict__ out, int64_t ldo,
                      int out_f32, int act, float* __restrict__ absmax, int M, int N, int K) {
    __shared__ float part[2][SK_WARPS][SK_NT][WIDE ? 16 : 8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;
    // Byte-balanced split: CTA i owns the contiguous output columns [N*i/G, N*(i+1)/G) — with G = 2 x SM count every
    // SM streams the same number of weight rows (to within one), whatever N is; the range is walked in MMA tiles
    // of 16 rows with the rows beyond the range masked off (not loaded).
    const int c_lo = (int)(((int64_t)N * blockIdx.x) / gridDim.x);
    const int c_hi = (int)(((int64_t)N * (blockIdx.x + 1)) / gridDim.x);
    const int nchunks = (K + 31) / 32;
    const int per_warp = (nchunks + SK_WARPS - 1) / SK_WARPS;
    const int c_begin = warp * per_warp, c_end = min(nchunks, c_begin + per_warp);
    const bool x_ok = g < M, x2_ok = WIDE && g + 8 < M;
    const __nv_bfloat16* xrow = x + (size_t)g * ldx + q * 8;
    const __nv_bfloat16* xrow2 = x + (size_t)(x2_ok ? g + 8 : g) * ldx + q * 8;
    const uint4 zero = make_uint4(0, 0, 0, 0);
    const uint64_t pol = make_evict_first_policy();
    float tmax = 0.f;
    bool waited = false;
    int buf = 0;
    for (int n0 = c_lo; n0 < c_hi; n0 += SK_NT, buf ^= 1) {
        const bool r0_ok = n0 + g < c_hi, r1_ok = n0 + g + 8 < c_hi;
        const __nv_bfloat16* wrow0 = W + (size_t)(n0 + g) * ldw + q * 8;
        const __nv_bfloat16* wrow1 = W + (size_t)(n0 + g + 8) * ldw + q * 8;
        auto load_w = [&](int c0, SkStage<UNROLL, WIDE>& st) {
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const int c = c0 + u;
                const bool in = c < c_end && c * 32 + q * 8 < K;
                st.w0[u] = (in && r0_ok) ? ld_stream(wrow0 + (size_t)c * 32, pol) : zero;
                st.w1[u] = (in && r1_ok) ? ld_stream(wrow1 + (size_t)c * 32, pol) : zero;
            }
        };
        auto load_x = [&](int c0, SkStage<UNROLL, WIDE>& st) {
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const int c = c0 + u;
                const bool in = c < c_end && c * 32 + q * 8 < K;
                st.xv[u] = (in && x_ok) ? *reinterpret_cast<const uint4*>(xrow + (size_t)c * 32) : zero;
                if (WIDE) st.xw[u] = (in && x2_ok) ? *reinterpret_cast<const uint4*>(xrow2 + (size_t)c * 32) : zero;
            }
        };
        float d[4] = {0.f, 0.f, 0.f, 0.f}, e[4] = {0.f, 0.f, 0.f, 0.f};
        SkStage<UNROLL, WIDE> st;
        // weights do not depend on the previous kernel: request them, let the next kernel start its own prologue,
        // and only then wait for the producer of x
        load_w(c_begin, st);
        if (!waited) {
            pdl_launch_dependents();
            pdl_wait();
            waited = true;
        }
        load_x(c_begin, st);
        // rolling prefetch: slot u is refilled with chunk c + SK_UNROLL + u right after it has been consumed, so each
        // warp keeps SK_UNROLL chunks (512 B of each of its 16 weight rows) in flight from one register set
        for (int c = c_begin; c < c_end; c += UNROLL) {
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                mma_bf16_16816(d, st.w0[u].x, st.w1[u].x, st.w0[u].y, st.w1[u].y, st.xv[u].x, st.xv[u].y);
                mma_bf16_16816(d, st.w0[u].z, st.w1[u].z, st.w0[u].w, st.w1[u].w, st.xv[u].z, st.xv[u].w);
                if (WIDE) {
                    mma_bf16_16816(e, st.w0[u].x, st.w1[u].x, st.w0[u].y, st.w1[u].y, st.xw[u].x, st.xw[u].y);
                    mma_bf16_16816(e, st.w0[u].z, st.w1[u].z, st.w0[u].w, st.w1[u].w, st.xw[u].z, st.xw[u].w);
                }
                const int cn = c + UNROLL + u;
                const bool in = cn < c_end && cn * 32 + q * 8 < K;
                st.w0[u] = (in && r0_ok) ? ld_stream(wrow0 + (size_t)cn * 32, pol) : zero;
                st.w1[u] = (in && r1_ok) ? ld_stream(wrow1 + (size_t)cn * 32, pol) : zero;
                st.xv[u] = (in && x_ok) ? *reinterpret_cast<const uint4*>(xrow + (size_t)cn * 32) : zero;
                if (WIDE) st.xw[u] = (in && x2_ok) ? *reinterpret_cast<const uint4*>(xrow2 + (size_t)cn * 32) : zero;
            }
        }
        // D fragment: d0,d1 = (row g, cols 2q,2q+1), d2,d3 = (row g+8, cols 2q,2q+1); row = output column, col = m
        part[buf][warp][g][2 * q] = d[0];
        part[buf][warp][g][2 * q + 1] = d[1];
        part[buf][warp][g + 8][2 * q] = d[2];
        part[buf][warp][g + 8][2 * q + 1] = d[3];
        if (WIDE) {
            part[buf][warp][g][8 + 2 * q] = e[0];
            part[buf][warp][g][8 + 2 * q + 1] = e[1];
            part[buf][warp][g + 8][8 + 2 * q] = e[2];
            part[buf][warp][g + 8][8 + 2 * q + 1] = e[3];
        }
        __syncthreads();
        if (threadIdx.x < SK_NT * (WIDE ? 16 : 8)) {
            const int m = threadIdx.x >> 4, nn = threadIdx.x & 15;   // consecutive threads -> consecutive columns
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < SK_WARPS; ++w) v += part[buf][w][nn][m];
            const int n = n0 + nn;
            if (m < M && n < c_hi) {
                if (bias != nullptr) v += __bfloat162float(bias[n]);
                if (act == 1) v = gelu_tanh(v);
                if (out_f32) {
                    static_cast<float*>(out)[(size_t)m * ldo + n] = v;
                    tmax = fmaxf(tmax, fabsf(v));
                } else {
                    const __nv_bfloat16 o = __float2bfloat16_rn(v);
                    static_cast<__nv_bfloat16*>(out)[(size_t)m * ldo + n] = o;
                    tmax = fmaxf(tmax, fabsf(__bfloat162float(o)));
                }
            }
        }
    }
    if (!waited) {       // empty column range: still take part in the launch chain
        pdl_launch_dependents();
        pdl_wait();
    }
    if (absmax != nullptr && warp < (WIDE ? 8 : 4)) {
        tmax = warp_max(tmax);
        if (lane == 0 && tmax > 0.f) atomic_max_nonneg(absmax, tmax);
    }
}

// ------------------------------------------------------------------------------------------------
// Sandwich-LN glue between two decode linears, one CTA for the whole [M, K] (M <= 16):
//   y  = res_in + LN_post(gemm_out / (max|gemm_out| / 8))       (third / fourth LayerNorm + residual add)
//   xn = LN_pre(y / (max|y| / 8))                               (post-attention / next input / final LayerNorm)
// mpu/sparse_transformer.py:326-331 and :337-340 + :319 of the next layer; max|y| is taken inside the CTA
// (the whole tensor is here), max|gemm_out| comes from the linear kernel that produced it.
// ------------------------------------------------------------------------------------------------
constexpr int LP_THREADS = 1024;
// MT: padded row count (warps are split evenly over the rows); NP: bf16 pairs per thread (K <= 2 * NP * threads/row)
template <int MT, int NP>
__global__ void __launch_bounds__(LP_THREADS)
ln_pair_kernel(const float* __restrict__ res_in, const __nv_bfloat16* __restrict__ gemm_out,
               const float* __restrict__ absmax_gemm, const __nv_bfloat16* __restrict__ g_post,
               const __nv_bfloat16* __restrict__ b_post, const __nv_bfloat16* __restrict__ g_pre,
               const __nv_bfloat16* __restrict__ b_pre, float eps, float* __restrict__ res_out,
               __nv_bfloat16* __restrict__ xn_out, int M, int K) {
    constexpr int WPR = 32 / MT;               // warps per row
    constexpr int TPR = WPR * 32;              // threads per row
    __shared__ float red[4][MT][WPR];
    __shared__ float smax[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = warp / WPR, wr = warp % WPR;
    const int tr = wr * 32 + lane;             // thread index within the row group
    const bool row_ok = row < M;
    const bool has_post = gemm_out != nullptr;

    // LayerNorm parameters are static: fetch them (packed bf16x2) before waiting for the producer kernel
    uint32_t gq[NP], bq[NP], gp[NP], bp[NP];
#pragma unroll
    for (int e = 0; e < NP; ++e) {
        const int k = 2 * (tr + e * TPR);
        const bool ok = k < K;
        gq[e] = ok ? *reinterpret_cast<const uint32_t*>(g_pre + k) : 0u;
        bq[e] = ok ? *reinterpret_cast<const uint32_t*>(b_pre + k) : 0u;
        gp[e] = (ok && has_post) ? *reinterpret_cast<const uint32_t*>(g_post + k) : 0u;
        bp[e] = (ok && has_post) ? *reinterpret_cast<const uint32_t*>(b_post + k) : 0u;
    }
    pdl_launch_dependents();
    pdl_wait();

    auto row_reduce = [&](float s, int buf) -> float {   // sum over the row group; one barrier per call
        s = warp_sum(s);
        if (lane == 0) red[buf][row][wr] = s;
        __syncthreads();
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < WPR; ++i) t += red[buf][row][i];
        return t;
    };
    auto lo = [](uint32_t u) { return __uint_as_float(u << 16); };
    auto hi = [](uint32_t u) { return __uint_as_float(u & 0xffff0000u); };

    float2 v[NP];
    const float inv_k = 1.0f / K;
    if (has_post) {
        uint32_t go[NP];
        float2 rs[NP];
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            const int k = 2 * (tr + e * TPR);
            const bool ok = k < K && row_ok;
            go[e] = ok ? *reinterpret_cast<const uint32_t*>(gemm_out + (size_t)row * K + k) : 0u;
            rs[e] = ok ? *reinterpret_cast<const float2*>(res_in + (size_t)row * K + k) : make_float2(0.f, 0.f);
        }
        const float c = *absmax_gemm * 0.125f;
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < NP; ++e) { v[e] = make_float2(lo(go[e]), hi(go[e])); s += v[e].x + v[e].y; }
        const float mean = row_reduce(s, 0) * inv_k;
        float ss = 0.f;
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            if (2 * (tr + e * TPR) < K) {
                const float a = v[e].x - mean, b = v[e].y - mean;
                ss += a * a + b * b;
            }
        }
        const float var = row_reduce(ss, 1) * inv_k;
        const float rstd = rsqrtf(var + eps * c * c);
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            v[e].x = (v[e].x - mean) * rstd * lo(gp[e]) + lo(bp[e]) + rs[e].x;
            v[e].y = (v[e].y - mean) * rstd * hi(gp[e]) + hi(bp[e]) + rs[e].y;
        }
    } else {
#pragma unroll
        for (int e = 0; e < NP; ++e) {
            const int k = 2 * (tr + e * TPR);
            v[e] = (k < K && row_ok) ? *reinterpret_cast<const float2*>(res_in + (size_t)row * K + k)
                                     : make_float2(0.f, 0.f);
        }
    }
    float mx = 0.f, s = 0.f;
#pragma unroll
    for (int e = 0; e < NP; ++e) {
        const int k = 2 * (tr + e * TPR);
        if (k < K && row_ok) {
            if (res_out != nullptr) *reinterpret_cast<float2*>(res_out + (size_t)row * K + k) = v[e];
            mx = fmaxf(mx, fmaxf(fabsf(v[e].x), fabsf(v[e].y)));
            s += v[e].x + v[e].y;
        }
    }
    mx = warp_max(mx);
    s = warp_sum(s);
    if (lane == 0) { smax[warp] = mx; red[2][row][wr] = s; }
    __syncthreads();
    float am = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) am = fmaxf(am, smax[i]);
    float tsum = 0.f;
#pragma unroll
    for (int i = 0; i < WPR; ++i) tsum += red[2][row][i];
    const float mean = tsum * inv_k;
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < NP; ++e) {
        if (2 * (tr + e * TPR) < K && row_ok) {
            const float a = v[e].x - mean, b = v[e].y - mean;
            ss += a * a + b * b;
        }
    }
    const float var = row_reduce(ss, 3) * inv_k;
    const float c = am * 0.125f;
    const float rstd = rsqrtf(var + eps * c * c);
#pragma unroll
    for (int e = 0; e < NP; ++e) {
        const int k = 2 * (tr + e * TPR);
        if (k < K && row_ok) {
            const float a = (v[e].x - mean) * rstd * lo(gq[e]) + lo(bq[e]);
            const float b = (v[e].y - mean) * rstd * hi(gq[e]) + hi(bq[e]);
            *reinterpret_cast<uint32_t*>(xn_out + (size_t)row * K + k) = pack_bf16x2(a, b);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// decode attention
// ------------------------------------------------------------------------------------------------
constexpr int DA_WARPS = 4;
constexpr int DA_UNROLL = 4;      // key blocks (of 16) in flight per CTA iteration
constexpr int HD = 64;

struct DecodeParams {
    const __nv_bfloat16* qkv;   // [b, 3h]: q | k_new | v_new of the token at position cur_len
    __nv_bfloat16* cache;       // [b, max_len, 2h]: K | V
    int64_t cache_bs;           // batch stride (elements)
    const int* cur_len_dev;     // device int32: number of cached tokens BEFORE this step (or null -> cur_len)
    int cur_len;
    __nv_bfloat16* out;         // [b, h]
    float* partial;             // [b, heads, nsplit, HD + 2] when nsplit > 1
    int heads, nsplit, max_len;
    float scale_log2;
    // GATHER (sparse_attention_inference, mpu/sparse_transformer.py:727-750, for sq = 1): the key set is the index list
    // idx[batch][0 .. *n_dev) (pivots + trailing window, the new token's position cur_len among them) instead of 0..t
    const int* idx;
    int64_t idx_bs;
    const int* n_dev;
    // RAGGED: row b holds *cur_len_dev - row_pad[b] cached tokens (0 <= row_pad[b] <= *cur_len_dev)
    const int* row_pad;
};

// 8 lanes cooperate on one key (8 dims each); a warp covers 4 keys per iteration.
// RAGGED: every row has its own t; the split-K ranges below follow from it, so a split may be empty for short rows.
template <bool GATHER, bool RAGGED>
__global__ void __launch_bounds__(DA_WARPS * 32)
attn_decode_kernel(const DecodeParams p) {
    __shared__ float s_m[DA_WARPS * 4], s_l[DA_WARPS * 4];
    __shared__ float s_acc[DA_WARPS * 4][HD];
    const int head = blockIdx.x, batch = blockIdx.y, split = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = lane >> 3, sub = lane & 7;
    const int h = p.heads * HD;
    pdl_launch_dependents();
    pdl_wait();
    // cached tokens of this row; the new token sits at index t
    const int t = (p.cur_len_dev ? *p.cur_len_dev : p.cur_len) - (RAGGED ? p.row_pad[batch] : 0);
    const __nv_bfloat16* qrow = p.qkv + (size_t)batch * 3 * h + head * HD + sub * 8;
    float q[8];
    bf16x8_to_float(*reinterpret_cast<const uint4*>(qrow), q);
    const uint4 knew = *reinterpret_cast<const uint4*>(qrow + h);
    const uint4 vnew = *reinterpret_cast<const uint4*>(qrow + 2 * h);
    __nv_bfloat16* kbase = p.cache + (size_t)batch * p.cache_bs + head * HD + sub * 8;
    // append (one split does it; the values are also used straight from registers below)
    if (split == p.nsplit - 1 && warp == 0 && grp == 0 && t < p.max_len) {
        *reinterpret_cast<uint4*>(kbase + (size_t)t * 2 * h) = knew;
        *reinterpret_cast<uint4*>(kbase + (size_t)t * 2 * h + h) = vnew;
    }
    const int total = GATHER ? *p.n_dev : t + 1;                // keys 0..t, or the gathered list
    const int* my_idx = GATHER ? p.idx + (size_t)batch * p.idx_bs : nullptr;
    const int per = (total + p.nsplit - 1) / p.nsplit;
    const int j0 = split * per, j1 = min(total, j0 + per);
    float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    // DA_UNROLL x 16 keys per CTA iteration: all loads of a block are issued before any is used (the loop is bound
    // by DRAM latency otherwise: one dependent 128-byte K and V fetch per key), and the online-softmax rescale runs
    // once per block.  The trip count is warp-uniform (the shuffles need all 32 lanes); out-of-range keys score -inf.
    for (int jb = j0 + warp * 4; jb < j1; jb += DA_WARPS * 4 * DA_UNROLL) {
        uint4 kr[DA_UNROLL], vr[DA_UNROLL];
        bool valid[DA_UNROLL];
#pragma unroll
        for (int u = 0; u < DA_UNROLL; ++u) {
            const int jj = jb + u * DA_WARPS * 4 + grp;
            valid[u] = jj < j1;
            const int j = (GATHER && valid[u]) ? my_idx[jj] : jj;       // cache position of this key
            kr[u] = knew;
            vr[u] = vnew;
            if (valid[u] && j != t) {
                const __nv_bfloat16* kp = kbase + (size_t)j * 2 * h;
                kr[u] = __ldg(reinterpret_cast<const uint4*>(kp));
                vr[u] = __ldg(reinterpret_cast<const uint4*>(kp + h));
            }
        }
        float sc[DA_UNROLL];
        float mn = m;
#pragma unroll
        for (int u = 0; u < DA_UNROLL; ++u) {
            float kf[8];
            bf16x8_to_float(kr[u], kf);
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) s = fmaf(q[i], kf[i], s);
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            s += __shfl_xor_sync(0xffffffffu, s, 4);
            sc[u] = valid[u] ? s * p.scale_log2 : -INFINITY;
            mn = fmaxf(mn, sc[u]);
        }
        if (mn > -INFINITY) {                       // at least one key seen so far by this lane group
            const float alpha = exp2f(m - mn);      // m = -inf on the first block -> 0
            m = mn;
            l *= alpha;
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] *= alpha;
#pragma unroll
            for (int u = 0; u < DA_UNROLL; ++u) {
                const float pr = exp2f(sc[u] - mn); // -inf -> 0
                float vf[8];
                bf16x8_to_float(vr[u], vf);
                l += pr;
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[i] = fmaf(pr, vf[i], acc[i]);
            }
        }
    }
    // combine the 16 (warp, group) partial states through shared memory
    const int slot = warp * 4 + grp;
    if (sub == 0) { s_m[slot] = m; s_l[slot] = l; }
#pragma unroll
    for (int i = 0; i < 8; ++i) s_acc[slot][sub * 8 + i] = acc[i];
    __syncthreads();
    if (threadIdx.x < HD) {
        const int d = threadIdx.x;
        float M = -INFINITY;
        for (int sidx = 0; sidx < DA_WARPS * 4; ++sidx) M = fmaxf(M, s_m[sidx]);
        float L = 0.f, A = 0.f;
        for (int sidx = 0; sidx < DA_WARPS * 4; ++sidx) {
            const float w = (s_m[sidx] == -INFINITY) ? 0.f : exp2f(s_m[sidx] - M);
            L += s_l[sidx] * w;
            A += s_acc[sidx][d] * w;
        }
        if (p.nsplit == 1) {
            p.out[(size_t)batch * h + head * HD + d] = __float2bfloat16_rn(A / L);
        } else {
            float* dst = p.partial + (((size_t)batch * p.heads + head) * p.nsplit + split) * (HD + 2);
            dst[d] = A;
            if (d == 0) { dst[HD] = M; dst[HD + 1] = L; }
        }
    }
}

__global__ void attn_decode_combine_kernel(const float* __restrict__ partial, __nv_bfloat16* __restrict__ out,
                                           int heads, int nsplit) {
    pdl_launch_dependents();
    pdl_wait();
    const int head = blockIdx.x, batch = blockIdx.y, d = threadIdx.x;
    const float* src = partial + ((size_t)batch * heads + head) * nsplit * (HD + 2);
    float M = -INFINITY;
    for (int s = 0; s < nsplit; ++s) M = fmaxf(M, src[s * (HD + 2) + HD]);
    float L = 0.f, A = 0.f;
    for (int s = 0; s < nsplit; ++s) {
        const float ms = src[s * (HD + 2) + HD];
        const float w = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
        L += src[s * (HD + 2) + HD + 1] * w;
        A += src[s * (HD + 2) + d] * w;
    }
    out[(size_t)batch * heads * HD + head * HD + d] = __float2bfloat16_rn(A / L);
}


// ------------------------------------------------------------------------------------------------
// Attention over a gathered key set (sparse_attention_inference, /root/reference/mpu/sparse_transformer.py:727-750):
// softmax((q / sqrt(hn)) K[idx]^T + causal(-10000 above the diagonal of the last sq x sq block)) V[idx].
// One CTA per (head, batch, query); keys come from the K|V cache through the index list (pivots U window).
// ------------------------------------------------------------------------------------------------
struct GatherParams {
    const __nv_bfloat16* q;     // [b, sq, h] view
    int64_t ldq, bsq;
    const __nv_bfloat16* cache; // [b, max_len, 2h]
    int64_t cache_bs;
    const int64_t* idx;         // [b, n]
    __nv_bfloat16* out;         // [b, sq, h] contiguous
    int heads, sq, n;
    float scale_log2;
};

__global__ void __launch_bounds__(DA_WARPS * 32)
attn_gather_kernel(const GatherParams p) {
    __shared__ float s_m[DA_WARPS * 4], s_l[DA_WARPS * 4];
    __shared__ float s_acc[DA_WARPS * 4][HD];
    const int head = blockIdx.x, batch = blockIdx.y, qi = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = lane >> 3, sub = lane & 7;
    const int h = p.heads * HD;
    float q[8];
    bf16x8_to_float(*reinterpret_cast<const uint4*>(p.q + (size_t)batch * p.bsq + (size_t)qi * p.ldq + head * HD + sub * 8), q);
    const __nv_bfloat16* kbase = p.cache + (size_t)batch * p.cache_bs + head * HD + sub * 8;
    const int64_t* idx = p.idx + (size_t)batch * p.n;
    const float masked = -10000.0f * 1.4426950408889634f;
    float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int jb = warp * 4; jb < p.n; jb += DA_WARPS * 4) {
        const int j = jb + grp;
        const bool valid = j < p.n;
        float kf[8], vf[8];
        if (valid) {
            const __nv_bfloat16* kp = kbase + (size_t)idx[j] * 2 * h;
            bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(kp)), kf);
            bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(kp + h)), vf);
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) { kf[i] = 0.f; vf[i] = 0.f; }
        }
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) s = fmaf(q[i], kf[i], s);
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        if (valid) {
            s *= p.scale_log2;
            const int rel = j - (p.n - p.sq);          // position inside the trailing query block
            if (p.sq > 1 && rel > qi) s += masked;    // scores + (-10000) above the diagonal (:741-745)
            const float mn = fmaxf(m, s);
            const float alpha = exp2f(m - mn), pr = exp2f(s - mn);
            m = mn;
            l = l * alpha + pr;
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = acc[i] * alpha + pr * vf[i];
        }
    }
    const int slot = warp * 4 + grp;
    if (sub == 0) { s_m[slot] = m; s_l[slot] = l; }
#pragma unroll
    for (int i = 0; i < 8; ++i) s_acc[slot][sub * 8 + i] = acc[i];
    __syncthreads();
    if (threadIdx.x < HD) {
        const int d = threadIdx.x;
        float M = -INFINITY;
        for (int sidx = 0; sidx < DA_WARPS * 4; ++sidx) M = fmaxf(M, s_m[sidx]);
        float L = 0.f, A = 0.f;
        for (int sidx = 0; sidx < DA_WARPS * 4; ++sidx) {
            const float w = (s_m[sidx] == -INFINITY) ? 0.f : exp2f(s_m[sidx] - M);
            L += s_l[sidx] * w;
            A += s_acc[sidx][d] * w;
        }
        p.out[((size_t)batch * p.sq + qi) * h + head * HD + d] = __float2bfloat16_rn(A / L);
    }
}

}  // namespace

extern "C" int cv_linear_small_m(const void* x, int64_t ldx, const void* W, int64_t ldw, const void* bias, void* out,
                                 int64_t ldo, int out_is_f32, int act, float* absmax, int M, int N, int K,
                                 void* stream) {
    CV_REQUIRE(x && W && out, "null pointer");
    CV_REQUIRE(M >= 1 && M <= 16, "cv_linear_small_m handles 1 <= M <= 16 rows (use cv_gemm_bf16 above that)");
    CV_REQUIRE(N > 0 && K > 0 && K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "K, ldx, ldw must be multiples of 8");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
               "x and W must be 16-byte aligned");
    CV_REQUIRE(act == 0 || act == 1, "act must be 0 or 1");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int grid = 2 * cvh::num_sms();                       // byte-balanced column ranges, two CTAs per SM
    if (grid > (N + 7) / 8) grid = (N + 7) / 8;          // tiny N: at least ~8 columns per CTA
    const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
    const __nv_bfloat16* wb = static_cast<const __nv_bfloat16*>(W);
    const __nv_bfloat16* bb = static_cast<const __nv_bfloat16*>(bias);
    // the MMA N dimension holds 8 batch rows: M <= 8 -> one B fragment set; 9..16 rows -> the WIDE kernel (two sets)
    if (M > 8) {
        CV_CUDA(cvh::launch_pdl(linear_small_m_kernel<SK_UNROLL / 2, true>, dim3(grid), dim3(SK_WARPS * 32), 0, s, true, xb,
                                ldx, wb, ldw, bb, out, ldo, out_is_f32, act, absmax, M, N, K));
        cvh::count_launches(1);
        return 0;
    }
    CV_CUDA(cvh::launch_pdl(linear_small_m_kernel<SK_UNROLL, false>, dim3(grid), dim3(SK_WARPS * 32), 0, s, true, xb, ldx,
                            wb, ldw, bb, out, ldo, out_is_f32, act, absmax, M, N, K));
    cvh::count_launches(1);
    return 0;
}

extern "C" int cv_ln_pair_small_m(const float* res_in, const void* gemm_out, const float* absmax_gemm,
                                  const void* g_post, const void* b_post, const void* g_pre, const void* b_pre,
                                  float eps, float* res_out, void* xn_out, int M, int K, void* stream) {
    CV_REQUIRE(res_in && g_pre && b_pre && xn_out, "null pointer");
    CV_REQUIRE(gemm_out == nullptr || (absmax_gemm && g_post && b_post), "gemm_out needs absmax_gemm, g_post, b_post");
    CV_REQUIRE(M >= 1 && M <= 16 && K > 0 && K % 2 == 0, "1 <= M <= 16, K even");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const __nv_bfloat16* go = static_cast<const __nv_bfloat16*>(gemm_out);
    const __nv_bfloat16 *gp = static_cast<const __nv_bfloat16*>(g_post), *bp = static_cast<const __nv_bfloat16*>(b_post);
    const __nv_bfloat16 *gq = static_cast<const __nv_bfloat16*>(g_pre), *bq = static_cast<const __nv_bfloat16*>(b_pre);
    __nv_bfloat16* xo = static_cast<__nv_bfloat16*>(xn_out);
    const int MT = M == 1 ? 1 : (M == 2 ? 2 : (M <= 4 ? 4 : (M <= 8 ? 8 : 16)));
    const int tpr = (32 / MT) * 32;
    const int need = (K + 2 * tpr - 1) / (2 * tpr);      // bf16 pairs per thread
    CV_REQUIRE(need <= 40, "K too large for cv_ln_pair_small_m at this M");
#define LP(MT_, NP_)                                                                                            \
    CV_CUDA(cvh::launch_pdl(ln_pair_kernel<MT_, NP_>, dim3(1), dim3(LP_THREADS), 0, s, true, res_in, go, absmax_gemm, \
                            gp, bp, gq, bq, eps, res_out, xo, M, K))
#define LP_BY_NP(MT_)                                  \
    do {                                               \
        if (need <= 2) LP(MT_, 2);                     \
        else if (need <= 5) LP(MT_, 5);                \
        else if (need <= 10) LP(MT_, 10);              \
        else if (need <= 20) LP(MT_, 20);              \
        else LP(MT_, 40);                              \
    } while (0)
    if (MT == 1) LP_BY_NP(1);
    else if (MT == 2) LP_BY_NP(2);
    else if (MT == 4) LP_BY_NP(4);
    else if (MT == 8) LP_BY_NP(8);
    else LP_BY_NP(16);
#undef LP_BY_NP
#undef LP
    cvh::count_launches(1);
    return 0;
}

extern "C" int64_t cv_attn_decode_workspace_bytes(int b, int heads, int nsplit) {
    return (int64_t)b * heads * nsplit * (HD + 2) * sizeof(float);
}

namespace {
// cv_attn_decode and cv_attn_decode_gather: attn_decode_kernel over the keys 0..t (idx == nullptr; RAGGED when
// row_pad is non-null) or over the gathered list idx (GATHER), then, for nsplit > 1, the split-K combine kernel.
int attn_decode_launch(const void* qkv, void* cache, int64_t cache_batch_stride, const int* cur_len_dev, int cur_len,
                       const int* row_pad, const int* idx, int64_t idx_batch_stride, const int* n_dev, void* out,
                       float* workspace, int b, int heads, int head_dim, int max_len, int nsplit, void* stream) {
    CV_REQUIRE(qkv && cache && out, "null pointer");
    CV_REQUIRE(head_dim == HD, "head_dim must be 64");
    CV_REQUIRE(b > 0 && heads > 0 && max_len > 0 && nsplit >= 1 && nsplit <= 64, "bad sizes");
    CV_REQUIRE(nsplit == 1 || workspace != nullptr, "workspace required when nsplit > 1");
    CV_REQUIRE(cur_len_dev != nullptr || (cur_len >= 0 && cur_len < max_len), "cur_len out of range");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DecodeParams p;
    p.qkv = static_cast<const __nv_bfloat16*>(qkv);
    p.cache = static_cast<__nv_bfloat16*>(cache);
    p.cache_bs = cache_batch_stride;
    p.cur_len_dev = cur_len_dev;
    p.cur_len = cur_len;
    p.out = static_cast<__nv_bfloat16*>(out);
    p.partial = workspace;
    p.heads = heads; p.nsplit = nsplit; p.max_len = max_len;
    p.scale_log2 = (1.0f / sqrtf((float)head_dim)) * 1.4426950408889634f;
    p.idx = idx; p.idx_bs = idx_batch_stride; p.n_dev = n_dev;
    p.row_pad = row_pad;
    dim3 grid(heads, b, nsplit);
    if (idx != nullptr) {
        CV_CUDA(cvh::launch_pdl(attn_decode_kernel<true, false>, grid, dim3(DA_WARPS * 32), 0, s, true, p));
    } else if (row_pad != nullptr) {
        CV_CUDA(cvh::launch_pdl(attn_decode_kernel<false, true>, grid, dim3(DA_WARPS * 32), 0, s, true, p));
    } else {
        CV_CUDA(cvh::launch_pdl(attn_decode_kernel<false, false>, grid, dim3(DA_WARPS * 32), 0, s, true, p));
    }
    cvh::count_launches(1);
    if (nsplit > 1) {
        CV_CUDA(cvh::launch_pdl(attn_decode_combine_kernel, dim3(heads, b), dim3(HD), 0, s, true,
                                static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out), heads, nsplit));
        cvh::count_launches(1);
    }
    return 0;
}
}  // namespace

extern "C" int cv_attn_decode(const void* qkv, void* cache, int64_t cache_batch_stride, const int* cur_len_dev,
                              int cur_len, const int* row_pad, void* out, float* workspace, int b, int heads,
                              int head_dim, int max_len, int nsplit, void* stream) {
    return attn_decode_launch(qkv, cache, cache_batch_stride, cur_len_dev, cur_len, row_pad, nullptr, 0, nullptr, out,
                              workspace, b, heads, head_dim, max_len, nsplit, stream);
}

extern "C" int cv_attn_gather(const void* q, int64_t ldq, int64_t bsq, const void* cache, int64_t cache_batch_stride,
                              const int64_t* idx, void* out, int b, int heads, int head_dim, int sq, int n,
                              void* stream) {
    CV_REQUIRE(q && cache && idx && out, "null pointer");
    CV_REQUIRE(head_dim == HD, "head_dim must be 64");
    CV_REQUIRE(b > 0 && heads > 0 && sq > 0 && n >= sq, "need n >= sq > 0 (the last sq indices are the queries)");
    CV_REQUIRE(sq <= 65535 && b <= 65535, "grid dimension limit");
    GatherParams p;
    p.q = static_cast<const __nv_bfloat16*>(q); p.ldq = ldq; p.bsq = bsq;
    p.cache = static_cast<const __nv_bfloat16*>(cache); p.cache_bs = cache_batch_stride;
    p.idx = idx; p.out = static_cast<__nv_bfloat16*>(out);
    p.heads = heads; p.sq = sq; p.n = n;
    p.scale_log2 = (1.0f / sqrtf((float)head_dim)) * 1.4426950408889634f;
    attn_gather_kernel<<<dim3(heads, b, sq), DA_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(p);
    CV_LAUNCH_CHECK();
    return 0;
}


// ------------------------------------------------------------------------------------------------
// Sparse inference on the device (is_sparse == 2, mpu/sparse_transformer.py:498-520, :591-600): the index plan of one
// decode step for EVERY layer in one launch.  Per (layer, sequence): all text positions before the trailing window plus a
// uniformly random subset of the image positions before it (num_pivot entries in total), then the window.  The reference
// draws the subset with Python's random.sample per layer per token on the host;
// here every candidate gets a counter-based random key and the smallest keys win — the same distribution (a uniformly
// random k-subset, fresh per layer and token), a different random stream.  One 64-bit bitonic sort per CTA orders
// "text first (key 0), then images by random key"; the first num_pivot entries are the pivots.
// ------------------------------------------------------------------------------------------------
constexpr int SP_THREADS = 1024;
constexpr int SP_MAXPOS = 4096;

__device__ __forceinline__ uint32_t sp_hash(uint64_t seed, uint32_t t, uint32_t layer, uint32_t b, uint32_t pos) {
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * ((((uint64_t)t << 32) | pos) + 0x632BE59BD9B4E019ull * (((uint64_t)layer << 16) | b));
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (uint32_t)(z >> 33);          // 31 bits
}

__global__ void __launch_bounds__(SP_THREADS)
sparse_plan_kernel(const uint8_t* __restrict__ is_txt, int64_t txt_bs, const int* __restrict__ cur_len_dev, int b,
                   int window, double ratio, const unsigned long long* __restrict__ seed_dev, int* __restrict__ idx,
                   int nmax, int* __restrict__ n_dev, int* __restrict__ err) {
    __shared__ unsigned long long keys[SP_MAXPOS];
    __shared__ int s_cnt[16];
    const int layer = blockIdx.x, bb = blockIdx.y, tid = threadIdx.x;
    const int t = *cur_len_dev, key_length = t + 1;
    const int lb = max(0, key_length - window);
    if (tid < 16) s_cnt[tid] = 0;
    __syncthreads();
    // text count of every sequence before the window (the reference sizes the pivot set by the maximum, :508-510)
    for (int q = 0; q < b; ++q) {
        int c = 0;
        for (int pp = tid; pp < lb; pp += SP_THREADS) c += is_txt[(size_t)q * txt_bs + pp] ? 1 : 0;
        c = __reduce_add_sync(0xffffffffu, c);
        if ((tid & 31) == 0 && c) atomicAdd(&s_cnt[q], c);
    }
    __syncthreads();
    int max_txt = 0;
    for (int q = 0; q < b; ++q) max_txt = max(max_txt, s_cnt[q]);
    const int num_pivot = max_txt + (int)((double)(lb - max_txt) * ratio);
    const int n_win = key_length - lb;
    if (num_pivot + n_win > nmax || lb > SP_MAXPOS) {
        if (tid == 0 && err) atomicExch(err, 1);
        return;
    }
    int n2 = 1;
    while (n2 < lb) n2 <<= 1;
    const unsigned long long seed = *seed_dev;
    for (int pp = tid; pp < n2; pp += SP_THREADS) {
        unsigned long long k = ~0ull;
        if (pp < lb)
            k = is_txt[(size_t)bb * txt_bs + pp] ? (unsigned long long)pp
                                                : (((unsigned long long)(1u + sp_hash(seed, (uint32_t)t, layer, bb, pp))) << 32) | (unsigned)pp;
        keys[pp] = k;
    }
    __syncthreads();
    for (int k2 = 2; k2 <= n2; k2 <<= 1) {
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < n2; i += SP_THREADS) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = keys[i], c = keys[ixj];
                    const bool up = (i & k2) == 0;
                    if ((a > c) == up) { keys[i] = c; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
    int* out = idx + ((size_t)layer * b + bb) * nmax;
    for (int i = tid; i < num_pivot; i += SP_THREADS) out[i] = (int)(keys[i] & 0xffffffffull);
    for (int i = tid; i < n_win; i += SP_THREADS) out[num_pivot + i] = lb + i;
    if (layer == 0 && bb == 0 && tid == 0) *n_dev = num_pivot + n_win;
}

extern "C" int cv_sparse_plan(const void* is_txt, int64_t txt_batch_stride, const int* cur_len_dev, int num_layers,
                              int b, int window, int num_pivot, int max_sequence_length, const void* seed_dev, int* idx,
                              int nmax, int* n_dev, int* err, void* stream) {
    CV_REQUIRE(is_txt && cur_len_dev && seed_dev && idx && n_dev, "null pointer");
    CV_REQUIRE(num_layers > 0 && b > 0 && b <= 16 && window > 0 && num_pivot >= 0 && max_sequence_length > 0 && nmax > 0,
               "bad sizes (batch <= 16)");
    sparse_plan_kernel<<<dim3(num_layers, b), SP_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint8_t*>(is_txt), txt_batch_stride, cur_len_dev, b, window,
        (double)num_pivot / (double)max_sequence_length, static_cast<const unsigned long long*>(seed_dev), idx, nmax, n_dev,
        err);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_attn_decode_gather(const void* qkv, void* cache, int64_t cache_batch_stride, const int* cur_len_dev,
                                     const int* idx, int64_t idx_batch_stride, const int* n_dev, void* out,
                                     float* workspace, int b, int heads, int head_dim, int max_len, int nsplit,
                                     void* stream) {
    CV_REQUIRE(cur_len_dev && idx && n_dev, "null pointer");
    return attn_decode_launch(qkv, cache, cache_batch_stride, cur_len_dev, -1, nullptr, idx, idx_batch_stride, n_dev,
                              out, workspace, b, heads, head_dim, max_len, nsplit, stream);
}
