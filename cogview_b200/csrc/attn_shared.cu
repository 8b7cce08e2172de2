// Single-token decode attention for rows that share a prompt (cv_attn_decode_shared): rows come in groups of G, the
// rows of a group are the beams of one prompt, and the prompt's K|V is held once per group in a prefix cache.  Row r
// of group g = r / G attends to prefix[g, 0:P], then to its own generated tokens suffix[r, 0:s], then to its new key,
// and appends its k|v at suffix[r, s].
//
// Image captioning is the shape it serves: a 1028-token image prompt and at most 20 generated text tokens per beam, 8
// beams per image.  Held as one cache row per beam, every step reads each prompt's K|V G times; here every prefix key
// and value is read from HBM ONCE per (group, head) for all G beams, as attn_chunk_kernel (csrc/attn_chunk.cu) reads
// each cached key once for all queries of a chunk.  One CTA owns one (head, group, prefix key range), stages 64-key K
// and V tiles in shared memory (cp.async, double-buffered), and the group's G queries consume them as 16-row
// mma.sync m16n8k16 tiles.  The prefix keys are split over gridDim.z CTAs so that a few groups still fill the SMs.
//
// A combine kernel per (row, head) then adds the row's own suffix keys and its new key on CUDA cores (a few dozen
// keys, different for every row), merges them with the partial softmax states of the prefix splits, and appends.
#include "common.cuh"
#include "mma_tile.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

constexpr int SH_HD = 64;          // head dim
constexpr int SH_WARPS = 4;        // 16 query rows per warp
constexpr int SH_MAXG = 16 * SH_WARPS;
constexpr int SH_KT = 64;          // keys per shared-memory tile
constexpr int SH_THREADS = SH_WARPS * 32;
constexpr int SH_CH = 128;         // suffix keys scored per pass of the combine kernel
constexpr int SH_PART = SH_HD + 2; // floats per partial state: o[64], m, l

struct SharedParams {
    const __nv_bfloat16* qkv;      // [b, 3h]: q | k_new | v_new
    const __nv_bfloat16* prefix;   // [groups, max_len, 2h]: K | V of the prompts (read only)
    int64_t prefix_bs;             // batch stride (elements)
    int P;                         // prefix length (every group)
    __nv_bfloat16* suffix;         // [b, s_max, 2h]: K | V of the generated tokens
    int64_t suffix_bs;
    const int* s_dev;              // suffix length on the device, or null: s
    int s;
    __nv_bfloat16* out;            // [b, h]
    float* partial;                // [b, heads, nsplit, HD + 2]
    int G, heads, nsplit;
    float scale_log2;
};

__global__ void __launch_bounds__(SH_THREADS)
attn_shared_prefix_kernel(const SharedParams p) {
    __shared__ __align__(128) __nv_bfloat16 s_q[SH_MAXG * SH_HD];
    __shared__ __align__(128) __nv_bfloat16 s_k[2][SH_KT * SH_HD];
    __shared__ __align__(128) __nv_bfloat16 s_v[2][SH_KT * SH_HD];
    const int head = blockIdx.x, grp = blockIdx.y, split = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, q4 = lane & 3;
    const int G = p.G, h = p.heads * SH_HD;
    const int per = ((p.P + p.nsplit - 1) / p.nsplit + SH_KT - 1) / SH_KT * SH_KT;
    const int j0 = split * per, j1 = min(p.P, j0 + per);
    const int ntiles = j1 > j0 ? (j1 - j0 + SH_KT - 1) / SH_KT : 0;
    const __nv_bfloat16* q_grp = p.qkv + (size_t)grp * G * 3 * h + head * SH_HD;          // beam i at + i * 3h
    const __nv_bfloat16* pre = p.prefix + (size_t)grp * p.prefix_bs + head * SH_HD;       // key j at + j * 2h

    // the group's queries (rows >= G zero-filled) and the first key tile
    for (int e = tid; e < SH_MAXG * 8; e += SH_THREADS) {
        const int r = e >> 3, c = e & 7;
        cp_async16(smem_u32(s_q) + swz(r, c), q_grp + (size_t)(r < G ? r : 0) * 3 * h + c * 8, r < G);
    }
    auto load_tile = [&](int jt, int st) {
        const uint32_t kb = smem_u32(s_k[st]), vb = smem_u32(s_v[st]);
        for (int e = tid; e < SH_KT * 8; e += SH_THREADS) {
            const int r = e >> 3, c = e & 7;
            const int j = jt + r;
            const bool ok = j < j1;
            const __nv_bfloat16* src = pre + (size_t)(ok ? j : 0) * 2 * h + c * 8;
            cp_async16(kb + swz(r, c), src, ok);
            cp_async16(vb + swz(r, c), src + h, ok);
        }
    };
    if (ntiles > 0) load_tile(j0, 0);
    cp_async_commit();

    const bool active = warp * 16 < G;                   // warp-uniform: this warp has query rows
    uint32_t qa[4][4];
    float o[8][4];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[dt][e] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    for (int it = 0; it < ntiles; ++it) {
        const int st = it & 1;
        if (it + 1 < ntiles) load_tile(j0 + (it + 1) * SH_KT, st ^ 1);
        cp_async_commit();
        cp_async_wait1();
        __syncthreads();
        if (active) {
            if (it == 0) {
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, c = 2 * ks + (lane >> 4);
                    ldsm_x4(smem_u32(s_q) + swz(r, c), qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3]);
                }
            }
            const uint32_t kb = smem_u32(s_k[st]), vb = smem_u32(s_v[st]);
            const int jt = j0 + it * SH_KT;
            // S = Q K^T over the tile's 64 keys (n-tile nt = keys 8nt .. 8nt+7)
            float s[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
                for (int kp = 0; kp < 2; ++kp) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4(kb + swz(8 * nt + (lane & 7), 4 * kp + (lane >> 3)), b0, b1, b2, b3);
                    mma16816(s[nt], qa[2 * kp], b0, b1);
                    mma16816(s[nt], qa[2 * kp + 1], b2, b3);
                }
            }
            // range mask, scale, online softmax (rows g and g + 8 of this warp; a quad shares a row)
            float mx0 = m0, mx1 = m1;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const bool ok = jt + 8 * nt + 2 * q4 + e < j1;
                    s[nt][e] = ok ? s[nt][e] * p.scale_log2 : -INFINITY;
                    s[nt][2 + e] = ok ? s[nt][2 + e] * p.scale_log2 : -INFINITY;
                    mx0 = fmaxf(mx0, s[nt][e]);
                    mx1 = fmaxf(mx1, s[nt][2 + e]);
                }
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            const float al0 = exp2f(m0 - mx0), al1 = exp2f(m1 - mx1);      // m = -inf -> 0 (every tile has a key)
            m0 = mx0;
            m1 = mx1;
            l0 *= al0;
            l1 *= al1;
#pragma unroll
            for (int dt = 0; dt < 8; ++dt) {
                o[dt][0] *= al0; o[dt][1] *= al0;
                o[dt][2] *= al1; o[dt][3] *= al1;
            }
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                s[nt][0] = exp2f(s[nt][0] - mx0);
                s[nt][1] = exp2f(s[nt][1] - mx0);
                s[nt][2] = exp2f(s[nt][2] - mx1);
                s[nt][3] = exp2f(s[nt][3] - mx1);
                l0 += s[nt][0] + s[nt][1];
                l1 += s[nt][2] + s[nt][3];
            }
            // O += P V: the C fragments of two key n-tiles are the A fragment of one 16-key step
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                uint32_t pa[4];
                pa[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
                pa[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
                pa[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
                pa[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
                for (int dp = 0; dp < 4; ++dp) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4_t(vb + swz(16 * kk + (lane & 7) + ((lane >> 3) & 1) * 8, 2 * dp + (lane >> 4)), b0, b1, b2, b3);
                    mma16816(o[2 * dp], pa, b0, b1);
                    mma16816(o[2 * dp + 1], pa, b2, b3);
                }
            }
        }
        __syncthreads();                                  // the next iteration refills this stage
    }

    if (!active) return;
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    // unnormalised partial state of every beam: an empty key range leaves o = 0, m = -inf, l = 0
    const int qi0 = warp * 16 + g, qi1 = qi0 + 8;
    const size_t r0 = (size_t)grp * G + qi0, r1 = r0 + 8;
    float* base0 = p.partial + ((r0 * p.heads + head) * p.nsplit + split) * SH_PART;
    float* base1 = p.partial + ((r1 * p.heads + head) * p.nsplit + split) * SH_PART;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
        const int d = 8 * dt + 2 * q4;
        if (qi0 < G) *reinterpret_cast<float2*>(base0 + d) = make_float2(o[dt][0], o[dt][1]);
        if (qi1 < G) *reinterpret_cast<float2*>(base1 + d) = make_float2(o[dt][2], o[dt][3]);
    }
    if (q4 == 0) {
        if (qi0 < G) { base0[SH_HD] = m0; base0[SH_HD + 1] = l0; }
        if (qi1 < G) { base1[SH_HD] = m1; base1[SH_HD + 1] = l1; }
    }
}

// per (row, head): the prefix splits' partial states, then the row's suffix keys 0..s-1 and its new key; appends the
// new k|v at suffix slot s (no other CTA reads that slot: suffix keys are read below s, the new key from qkv)
__global__ void __launch_bounds__(SH_THREADS)
attn_shared_combine_kernel(const SharedParams p) {
    __shared__ float s_q[SH_HD];
    __shared__ float s_sc[SH_CH];
    const int head = blockIdx.x, row = blockIdx.y;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int h = p.heads * SH_HD;
    const int s = p.s_dev != nullptr ? *p.s_dev : p.s;
    const __nv_bfloat16* qkv_row = p.qkv + (size_t)row * 3 * h + head * SH_HD;
    __nv_bfloat16* suf = p.suffix + (size_t)row * p.suffix_bs + head * SH_HD;             // slot j at + j * 2h
    if (tid < SH_HD) s_q[tid] = __bfloat162float(qkv_row[tid]);
    if (tid < 16) {
        const int part = tid >> 3, c = tid & 7;                                           // part 0: K, 1: V
        *reinterpret_cast<uint4*>(suf + (size_t)s * 2 * h + part * h + c * 8) =
            *reinterpret_cast<const uint4*>(qkv_row + (part + 1) * h + c * 8);
    }
    const float* ps = p.partial + ((size_t)row * p.heads + head) * p.nsplit * SH_PART;
    float M = -INFINITY;
    for (int sp = 0; sp < p.nsplit; ++sp) M = fmaxf(M, ps[sp * SH_PART + SH_HD]);
    float L = 0.f, A = 0.f;                                                               // A: dim tid (< 64)
    for (int sp = 0; sp < p.nsplit; ++sp) {
        const float m = ps[sp * SH_PART + SH_HD];
        const float w = m == -INFINITY ? 0.f : exp2f(m - M);
        L += ps[sp * SH_PART + SH_HD + 1] * w;
        if (tid < SH_HD) A += ps[sp * SH_PART + tid] * w;
    }
    __syncthreads();
    for (int c0 = 0; c0 <= s; c0 += SH_CH) {
        const int n = min(SH_CH, s + 1 - c0);
        for (int jj = warp; jj < n; jj += SH_WARPS) {                                     // one key per warp
            const int j = c0 + jj;
            const __nv_bfloat16* kp = j < s ? suf + (size_t)j * 2 * h : qkv_row + h;
            const float2 kf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(kp + 2 * lane));
            const float d = warp_sum(s_q[2 * lane] * kf.x + s_q[2 * lane + 1] * kf.y);
            if (lane == 0) s_sc[jj] = d * p.scale_log2;
        }
        __syncthreads();
        float cm = M;
        for (int jj = 0; jj < n; ++jj) cm = fmaxf(cm, s_sc[jj]);
        const float al = exp2f(M - cm);                                                   // M = -inf -> 0
        M = cm;
        L *= al;
        A *= al;
        for (int jj = 0; jj < n; ++jj) {
            const int j = c0 + jj;
            const float w = exp2f(s_sc[jj] - M);
            L += w;
            if (tid < SH_HD) A += w * __bfloat162float(j < s ? suf[(size_t)j * 2 * h + h + tid] : qkv_row[2 * h + tid]);
        }
        __syncthreads();                                                                  // s_sc is refilled
    }
    if (tid < SH_HD) p.out[(size_t)row * h + head * SH_HD + tid] = __float2bfloat16_rn(A / L);
}

}  // namespace

extern "C" int64_t cv_attn_shared_workspace_bytes(int b, int heads, int nsplit) {
    return (int64_t)b * heads * nsplit * SH_PART * sizeof(float);
}

extern "C" int cv_attn_decode_shared(const void* qkv, const void* prefix, int64_t prefix_batch_stride, int prefix_len,
                                     int max_len, void* suffix, int64_t suffix_batch_stride, const int* s_dev, int s,
                                     int s_max, void* out, float* workspace, int b, int groups, int heads,
                                     int head_dim, int nsplit, void* stream) {
    CV_REQUIRE(qkv && prefix && suffix && out && workspace, "null pointer");
    CV_REQUIRE(head_dim == SH_HD, "head_dim must be 64");
    CV_REQUIRE(b > 0 && b <= 65535 && heads > 0 && heads <= 65535 && groups > 0, "bad sizes");
    CV_REQUIRE(b % groups == 0 && b / groups <= SH_MAXG, "rows must form groups of 1 <= G <= 64 (b % groups == 0)");
    CV_REQUIRE(prefix_len >= 0 && prefix_len <= max_len, "need 0 <= P <= max_len");
    CV_REQUIRE(s_max >= 1 && (s_dev != nullptr || (s >= 0 && s < s_max)), "need 0 <= s < s_max");
    CV_REQUIRE(nsplit >= 1 && nsplit <= 64, "1 <= nsplit <= 64");
    CV_REQUIRE(prefix_batch_stride >= (int64_t)max_len * 2 * heads * SH_HD &&
                   suffix_batch_stride >= (int64_t)s_max * 2 * heads * SH_HD,
               "batch strides below max_len * 2h / s_max * 2h");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(prefix) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(suffix) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && prefix_batch_stride % 8 == 0 &&
                   suffix_batch_stride % 8 == 0,
               "qkv, prefix, suffix, out and workspace must be 16-byte aligned, the batch strides multiples of 8");
    SharedParams p;
    p.qkv = static_cast<const __nv_bfloat16*>(qkv);
    p.prefix = static_cast<const __nv_bfloat16*>(prefix);
    p.prefix_bs = prefix_batch_stride;
    p.P = prefix_len;
    p.suffix = static_cast<__nv_bfloat16*>(suffix);
    p.suffix_bs = suffix_batch_stride;
    p.s_dev = s_dev;
    p.s = s;
    p.out = static_cast<__nv_bfloat16*>(out);
    p.partial = workspace;
    p.G = b / groups;
    p.heads = heads;
    p.nsplit = nsplit;
    p.scale_log2 = (1.0f / sqrtf((float)head_dim)) * 1.4426950408889634f;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    attn_shared_prefix_kernel<<<dim3(heads, groups, nsplit), SH_THREADS, 0, st>>>(p);
    CV_LAUNCH_CHECK();
    attn_shared_combine_kernel<<<dim3(heads, b), SH_THREADS, 0, st>>>(p);
    CV_LAUNCH_CHECK();
    return 0;
}
