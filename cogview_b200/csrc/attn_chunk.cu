// Ragged multi-token attention on the K|V cache (cv_attn_chunk_ragged): a chunk of n new tokens per sequence attends
// to that sequence's own cached prefix and to itself (causal inside the chunk), and the chunk's K|V is appended.
// It is the multi-query form of cv_attn_decode with row_pad (csrc/decode.cu): super-resolution templates interleave
// given stretches of codes with generated ones, and the given stretch plus the last sampled token (17 tokens) go
// through the model as one chunk for every image of a decode batch, each image at its own cache length.
//
// At the shapes it serves the kernel is bound by reading the cache (64 rows x ~1300 tokens x 5120 bf16 columns is
// ~0.85 GB per layer), so the design point is that every cached key and value is read from HBM ONCE per (row, head)
// for all n queries of the chunk: one CTA owns one (head, row, key range), stages 64-key K and V tiles in shared memory
// (cp.async, double-buffered) and all of its query rows consume them.  The key range of a row is split over
// gridDim.z CTAs (each row's ranges follow from its own key count) and a combine pass merges the partial softmax
// states, as attn_decode_kernel does, so that a small batch still fills the SMs.
//
// Tensor cores: warp-level mma.sync m16n8k16 (bf16 -> fp32), not wgmma.  The query dimension is small (17 for the
// callers, at most 64) and ragged: with mma.sync each warp owns 16 query rows, so 17 queries cost two warps' MMAs
// rather than a 64-row wgmma tile, and the K / V operands come straight from the XOR-swizzled tiles through
// ldmatrix (.trans for V).  The MMAs are far from the bound either way; what matters is the single pass over the cache.
#include "common.cuh"
#include "mma_tile.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

constexpr int CK_HD = 64;          // head dim
constexpr int CK_WARPS = 4;        // 16 query rows per warp
constexpr int CK_MAXN = 16 * CK_WARPS;
constexpr int CK_KT = 64;          // keys per shared-memory tile
constexpr int CK_THREADS = CK_WARPS * 32;

struct ChunkParams {
    const __nv_bfloat16* qkv;      // [b, n, 3h]: q | k | v of the chunk, token-major
    __nv_bfloat16* cache;          // [b, max_len, 2h]: K | V
    int64_t cache_bs;              // batch stride (elements)
    int cur_len;
    const int* row_pad;            // [b] or null: row r holds cur_len - row_pad[r] cached tokens
    __nv_bfloat16* out;            // [b, n, h]
    float* partial;                // [b, heads, nsplit, n, HD + 2] when nsplit > 1
    int n, heads, nsplit;
    float scale_log2;
};

__global__ void __launch_bounds__(CK_THREADS)
attn_chunk_kernel(const ChunkParams p) {
    __shared__ __align__(128) __nv_bfloat16 s_q[CK_MAXN * CK_HD];
    __shared__ __align__(128) __nv_bfloat16 s_k[2][CK_KT * CK_HD];
    __shared__ __align__(128) __nv_bfloat16 s_v[2][CK_KT * CK_HD];
    const int head = blockIdx.x, row = blockIdx.y, split = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, q4 = lane & 3;
    const int n = p.n, h = p.heads * CK_HD;
    const int t = p.cur_len - (p.row_pad != nullptr ? p.row_pad[row] : 0);   // cached tokens of this row
    const int total = t + n;                                                 // keys: the cache, then the chunk
    const int per = ((total + p.nsplit - 1) / p.nsplit + CK_KT - 1) / CK_KT * CK_KT;
    const int j0 = split * per, j1 = min(total, j0 + per);
    const int ntiles = j1 > j0 ? (j1 - j0 + CK_KT - 1) / CK_KT : 0;
    const __nv_bfloat16* qkv_row = p.qkv + (size_t)row * n * 3 * h + head * CK_HD;   // token i at + i * 3h
    __nv_bfloat16* cache_row = p.cache + (size_t)row * p.cache_bs + head * CK_HD;    // slot j at + j * 2h

    // append the chunk's K|V at slots t .. t+n-1.  One split writes; every split reads the chunk's keys from qkv, and
    // the cache slots it reads are all below t, so no CTA reads what another writes.
    if (split == 0) {
        for (int e = tid; e < n * 16; e += CK_THREADS) {
            const int i = e >> 4, part = (e >> 3) & 1, c = e & 7;              // part 0: K, 1: V
            const uint4 v = *reinterpret_cast<const uint4*>(qkv_row + (size_t)i * 3 * h + (part + 1) * h + c * 8);
            *reinterpret_cast<uint4*>(cache_row + (size_t)(t + i) * 2 * h + part * h + c * 8) = v;
        }
    }

    // queries (rows >= n zero-filled) and the first key tile
    for (int e = tid; e < CK_MAXN * 8; e += CK_THREADS) {
        const int r = e >> 3, c = e & 7;
        cp_async16(smem_u32(s_q) + swz(r, c), qkv_row + (size_t)(r < n ? r : 0) * 3 * h + c * 8, r < n);
    }
    auto load_tile = [&](int jt, int st) {
        const uint32_t kb = smem_u32(s_k[st]), vb = smem_u32(s_v[st]);
        for (int e = tid; e < CK_KT * 8; e += CK_THREADS) {
            const int r = e >> 3, c = e & 7;
            const int j = jt + r;
            const bool ok = j < j1;
            const __nv_bfloat16* src = j < t ? cache_row + (size_t)j * 2 * h + c * 8            // cached key j
                                             : qkv_row + (size_t)(ok ? j - t : 0) * 3 * h + h + c * 8;   // chunk key
            cp_async16(kb + swz(r, c), src, ok);
            cp_async16(vb + swz(r, c), src + h, ok);        // V follows K by h elements in both layouts
        }
    };
    if (ntiles > 0) load_tile(j0, 0);
    cp_async_commit();

    const bool active = warp * 16 < n;                   // warp-uniform: this warp has query rows
    const int lim0 = t + warp * 16 + g, lim1 = lim0 + 8; // last key visible to the C-fragment rows g and g + 8
    uint32_t qa[4][4];
    float o[8][4];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[dt][e] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    for (int it = 0; it < ntiles; ++it) {
        const int st = it & 1;
        if (it + 1 < ntiles) load_tile(j0 + (it + 1) * CK_KT, st ^ 1);
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
            const int jt = j0 + it * CK_KT;
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
            // causal + range mask, scale, online softmax (rows g and g + 8 of this warp; a quad shares a row)
            float mx0 = m0, mx1 = m1;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int j = jt + 8 * nt + 2 * q4 + e;
                    s[nt][e] = (j < j1 && j <= lim0) ? s[nt][e] * p.scale_log2 : -INFINITY;
                    s[nt][2 + e] = (j < j1 && j <= lim1) ? s[nt][2 + e] * p.scale_log2 : -INFINITY;
                    mx0 = fmaxf(mx0, s[nt][e]);
                    mx1 = fmaxf(mx1, s[nt][2 + e]);
                }
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            const float base0 = mx0 == -INFINITY ? 0.f : mx0, base1 = mx1 == -INFINITY ? 0.f : mx1;
            const float al0 = exp2f(m0 - base0), al1 = exp2f(m1 - base1);      // m = -inf -> 0
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
                s[nt][0] = exp2f(s[nt][0] - base0);
                s[nt][1] = exp2f(s[nt][1] - base0);
                s[nt][2] = exp2f(s[nt][2] - base1);
                s[nt][3] = exp2f(s[nt][3] - base1);
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
    const int qi0 = warp * 16 + g, qi1 = qi0 + 8;
    if (p.nsplit == 1) {
        const float inv0 = 1.f / l0, inv1 = 1.f / l1;
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) {
            const int d = head * CK_HD + 8 * dt + 2 * q4;
            if (qi0 < n)
                *reinterpret_cast<uint32_t*>(p.out + ((size_t)row * n + qi0) * h + d) = pack_bf16x2(o[dt][0] * inv0, o[dt][1] * inv0);
            if (qi1 < n)
                *reinterpret_cast<uint32_t*>(p.out + ((size_t)row * n + qi1) * h + d) = pack_bf16x2(o[dt][2] * inv1, o[dt][3] * inv1);
        }
    } else {
        float* base = p.partial + (((size_t)row * p.heads + head) * p.nsplit + split) * n * (CK_HD + 2);
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) {
            const int d = 8 * dt + 2 * q4;
            if (qi0 < n) *reinterpret_cast<float2*>(base + (size_t)qi0 * (CK_HD + 2) + d) = make_float2(o[dt][0], o[dt][1]);
            if (qi1 < n) *reinterpret_cast<float2*>(base + (size_t)qi1 * (CK_HD + 2) + d) = make_float2(o[dt][2], o[dt][3]);
        }
        if (q4 == 0) {
            if (qi0 < n) { base[(size_t)qi0 * (CK_HD + 2) + CK_HD] = m0; base[(size_t)qi0 * (CK_HD + 2) + CK_HD + 1] = l0; }
            if (qi1 < n) { base[(size_t)qi1 * (CK_HD + 2) + CK_HD] = m1; base[(size_t)qi1 * (CK_HD + 2) + CK_HD + 1] = l1; }
        }
    }
}

// merge the nsplit partial softmax states of every (row, head, query)
__global__ void __launch_bounds__(256)
attn_chunk_combine_kernel(const float* __restrict__ partial, __nv_bfloat16* __restrict__ out, int heads, int nsplit,
                          int n) {
    const int head = blockIdx.x, row = blockIdx.y;
    const float* src = partial + ((size_t)row * heads + head) * nsplit * n * (CK_HD + 2);
    for (int e = threadIdx.x; e < n * CK_HD; e += blockDim.x) {
        const int i = e / CK_HD, d = e % CK_HD;
        float M = -INFINITY;
        for (int s = 0; s < nsplit; ++s) M = fmaxf(M, src[((size_t)s * n + i) * (CK_HD + 2) + CK_HD]);
        float L = 0.f, A = 0.f;
        for (int s = 0; s < nsplit; ++s) {
            const float* ps = src + ((size_t)s * n + i) * (CK_HD + 2);
            const float w = (ps[CK_HD] == -INFINITY) ? 0.f : exp2f(ps[CK_HD] - M);
            L += ps[CK_HD + 1] * w;
            A += ps[d] * w;
        }
        out[((size_t)row * n + i) * heads * CK_HD + head * CK_HD + d] = __float2bfloat16_rn(A / L);
    }
}

}  // namespace

extern "C" int64_t cv_attn_chunk_workspace_bytes(int b, int heads, int n, int nsplit) {
    return (int64_t)b * heads * nsplit * n * (CK_HD + 2) * sizeof(float);
}

extern "C" int cv_attn_chunk_ragged(const void* qkv, void* cache, int64_t cache_batch_stride, int cur_len,
                                    const int* row_pad, void* out, float* workspace, int b, int n, int heads,
                                    int head_dim, int max_len, int nsplit, void* stream) {
    CV_REQUIRE(qkv && cache && out, "null pointer");
    CV_REQUIRE(head_dim == CK_HD, "head_dim must be 64");
    CV_REQUIRE(b > 0 && b <= 65535 && heads > 0 && heads <= 65535 && max_len > 0, "bad sizes");
    CV_REQUIRE(n >= 1 && n <= CK_MAXN, "the chunk holds 1 <= n <= 64 tokens");
    CV_REQUIRE(cur_len >= 0 && (int64_t)cur_len + n <= max_len, "need 0 <= cur_len and cur_len + n <= max_len");
    CV_REQUIRE(nsplit >= 1 && nsplit <= 64, "1 <= nsplit <= 64");
    CV_REQUIRE(nsplit == 1 || workspace != nullptr, "workspace required when nsplit > 1");
    CV_REQUIRE(cache_batch_stride >= (int64_t)max_len * 2 * heads * CK_HD, "cache batch stride below max_len * 2h");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(cache) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) & 15) == 0 && cache_batch_stride % 8 == 0,
               "qkv, cache and out must be 16-byte aligned, the cache batch stride a multiple of 8");
    ChunkParams p;
    p.qkv = static_cast<const __nv_bfloat16*>(qkv);
    p.cache = static_cast<__nv_bfloat16*>(cache);
    p.cache_bs = cache_batch_stride;
    p.cur_len = cur_len;
    p.row_pad = row_pad;
    p.out = static_cast<__nv_bfloat16*>(out);
    p.partial = workspace;
    p.n = n;
    p.heads = heads;
    p.nsplit = nsplit;
    p.scale_log2 = (1.0f / sqrtf((float)head_dim)) * 1.4426950408889634f;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    attn_chunk_kernel<<<dim3(heads, b, nsplit), CK_THREADS, 0, s>>>(p);
    CV_LAUNCH_CHECK();
    if (nsplit > 1) {
        attn_chunk_combine_kernel<<<dim3(heads, b), 256, 0, s>>>(workspace, p.out, heads, nsplit, n);
        CV_LAUNCH_CHECK();
    }
    return 0;
}
