// cv_attn_fwd: fused dense attention forward (flash-style, nothing of size [sq, sk] ever reaches HBM).
//
// Replaces standard_attention (/root/reference/mpu/sparse_transformer.py:652-673) together with the
// split / head-permute copies around it in GPT2ParallelSelfAttention.forward (:131-163):
//     softmax( (Q / sqrt(hn)) K^T * mask - 10000 * (1 - mask) ) V
// for the two mask families the reference builds: lower-triangular (pretrain_gpt2.py:218-221) and the
// int-`sep` form (mpu/sparse_transformer.py:477-489: keys [0, sep + mem) visible to every query, causal
// after that), with sq <= sk (queries are the LAST sq positions of the sk keys: decode-with-memory prefill).
// Masked scores are exactly -10000 as in the reference; whole key tiles that are masked for every query
// of the block are skipped (their softmax weight underflows to 0 in fp32).
//
// Q, K, V are read in place from the packed QKV GEMM output [b, s, 3h] (or a KV cache) through 3-D TMA
// tensor maps; the context is written token-major [b, sq, h] — the layout the out-projection GEMM reads.
//
// One CTA per (128-query block, head, batch); 3 warpgroups:
//   warpgroup 0     TMA producer (one thread): Q once, K/V tiles of 128 keys through a 3-stage ring
//   warpgroups 1-2  64 query rows each: S = Q K^T (wgmma m64n128k16, fp32 in registers), online softmax in registers
//                   (the four threads of a quad share a pair of rows), P as bf16 registers straight into the A operand
//                   of O += P V (m64n64k16).  The two warpgroups run independently, so the softmax of one overlaps
//                   the MMAs of the other.
#include "attention_sparse.cuh"
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

constexpr int BQ = 128;       // queries per CTA
constexpr int BKV = 128;      // keys per tile
constexpr int HD = 64;        // head dim (CogView: 2560 / 40)
constexpr int KV_STAGES = 3;
constexpr int Q_BYTES = BQ * HD * 2;        // 16 KB
constexpr int K_BYTES = BKV * HD * 2;       // 16 KB
constexpr int V_BYTES = BKV * HD * 2;       // 16 KB
constexpr int SMEM_BYTES = Q_BYTES + KV_STAGES * (K_BYTES + V_BYTES) + 1024 + 256;
constexpr int NUM_THREADS = 384;
constexpr float LOG2E = 1.4426950408889634f;

struct AttnParams {
    int b, heads, sq, sk;
    int sep_eff;        // keys [0, sep_eff) are visible to every query
    int off;            // sk - sq: query i sees key j <= i + off
    float scale_log2;   // (1/sqrt(hn)) * log2(e)
    __nv_bfloat16* out; // [b, sq, heads*HD]
    int64_t ldo;        // row stride of out (elements)
    int64_t bso;        // batch stride of out (elements)
    float* lse;         // [b, heads, sq] natural-log LSE, or null
    DropoutArgs drop;   // attention-probability dropout (mpu/sparse_transformer.py:667-669); p = 0 disables
    uint32_t* drop_mask;// two regions of b*heads*nkb_all*nqb_all*128 uint4 each, written by attn_dropout_mask_kernel:
                        //  [0] key-major [b, heads, nkb_all*128 (key), nqb_all, 4]: word w of (key, query block) holds
                        //      queries qb*128 + 32w .. +31 (what the backward consumes: one 16-byte load per key row)
                        //  [1] query-major [b, heads, nqb_all*128 (query), nkb_all, 4]: what this kernel consumes
                        // (sparse: the three regions of sparse::KeepLayout, written by attn_sparse_dropout_mask_kernel)
    const uint32_t* keep_q; // the query-major keep bits this kernel reads: [b, heads, nqb_all*128, keep_slots, 4]
    int keep_slots;         // entries per query row: nkb_all (dense), or one per tile of the sparse tile walk
    int nkb_all;        // ceil(sk / 128)
    int nqb_all;        // ceil(sq / 128)
    // sparse training attention (mpu/sparse_transformer.py:675-725; sp_w = 0: dense).  One softmax over
    //   band   : keys j with band_start(i) <= j <= i,  band_start(i) = max(0, i / sp_w - sp_times + 1) * sp_w
    //   pivots : gathered keys p with piv_pos[p] < band_start(i), score + log(s / n_piv)
    // (the closed form of the reference's window mask + rmask-gathered pivot mask, oracle/sparse_decomposition.py)
    int sp_w, sp_times, n_piv;
    const int* piv_pos;     // [b, n_piv] positions of the gathered pivot keys
    float piv_bias_log2;    // log(s / n_piv) * log2(e)
};

using sparse::band_start;

template <bool DROPOUT, bool SPARSE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmPK,
                const __grid_constant__ CUtensorMap tmPV, const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sKV = sQ + Q_BYTES;                              // stage s: K at s*(K+V), V after it
    uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + KV_STAGES * (K_BYTES + V_BYTES));
    uint64_t* q_full = bars;                 // [1]
    uint64_t* kv_full = bars + 1;            // [KV_STAGES]
    uint64_t* kv_empty = kv_full + KV_STAGES;// [KV_STAGES]: one arrive per consumer warp

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    // heaviest (last) query blocks first
    const int qb = gridDim.x - 1 - blockIdx.x;
    const int head = blockIdx.y, batch = blockIdx.z;
    const int q0 = qb * BQ;
    // number of key tiles any query of this block can see
    int kmax = q0 + BQ + p.off;              // exclusive bound of causally visible keys for the last row
    if (kmax < p.sep_eff) kmax = p.sep_eff;
    if (kmax > p.sk) kmax = p.sk;
    int nkb = (kmax + BKV - 1) / BKV;
    // sparse: band tiles jb0 .. jb0 + nband - 1 of the real keys first, then every pivot tile (if any query of the
    // block can see a pivot at all); one tile list for the three roles
    int jb0 = 0, nband = nkb;
    if (SPARSE) {
        const int q_last = min(q0 + BQ, p.sq) - 1;
        jb0 = band_start(q0, p.sp_w, p.sp_times) / BKV;
        nband = q_last / BKV - jb0 + 1;
        const int npt = band_start(q_last, p.sp_w, p.sp_times) > 0 ? (p.n_piv + BKV - 1) / BKV : 0;
        nkb = nband + npt;
    }

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        mbar_init(q_full, 1);
        for (int i = 0; i < KV_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tid == 0) {
            mbar_expect_tx(q_full, Q_BYTES);
            tma_load_3d(sQ, &tmQ, q_full, head * HD, q0, batch);
            int stage = 0; uint32_t phase = 0;
            for (int j = 0; j < nkb; ++j) {
                mbar_wait<false>(&kv_empty[stage], phase ^ 1);
                uint8_t* sK = sKV + stage * (K_BYTES + V_BYTES);
                mbar_expect_tx(&kv_full[stage], K_BYTES + V_BYTES);
                if (SPARSE && j >= nband) {
                    tma_load_3d(sK, &tmPK, &kv_full[stage], head * HD, (j - nband) * BKV, batch);
                    tma_load_3d(sK + K_BYTES, &tmPV, &kv_full[stage], head * HD, (j - nband) * BKV, batch);
                } else {
                    tma_load_3d(sK, &tmK, &kv_full[stage], head * HD, (jb0 + j) * BKV, batch);
                    tma_load_3d(sK + K_BYTES, &tmV, &kv_full[stage], head * HD, (jb0 + j) * BKV, batch);
                }
                if (++stage == KV_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ------------------------------ MMA + softmax warpgroups ------------------------------
        // Fragment layout (common.cuh): this thread holds rows r_loc and r_loc + 8 of the block, and of every
        // 8-column group the two columns c_in, c_in + 1.  Row statistics are reduced over the 4 lanes of a quad.
        setmaxnreg_inc<232>();
        const int half = wg - 1, warp = tid >> 5, lane = tid & 31;
        const int r_loc = 64 * half + 16 * warp + (lane >> 2);
        const int c_in = 2 * (lane & 3);
        int qi[2], causal_lim[2], bs_row[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            qi[h] = q0 + r_loc + 8 * h;                    // query index within the sequence
            causal_lim[h] = qi[h] + p.off;                 // last causally visible key
            bs_row[h] = SPARSE ? band_start(qi[h], p.sp_w, p.sp_times) : 0;
        }
        float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
        float o[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
        const float masked_val = -10000.0f * LOG2E;
        const uint4* keep_row[2] = {nullptr, nullptr};
        if (DROPOUT) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
                keep_row[h] = reinterpret_cast<const uint4*>(p.keep_q) +
                              (((size_t)batch * p.heads + head) * p.nqb_all * BQ + qi[h]) * p.keep_slots;
        }
        const uint32_t q_addr = smem_u32(sQ) + half * (64 * 128);
        mbar_wait<false>(q_full, 0);
        int stage = 0; uint32_t phase = 0;
        for (int j = 0; j < nkb; ++j) {
            // keep bits of this thread's 32 keys of rows h = 0, 1: bit 8 (i & 3) + 2 (i >> 2) + e <-> key 8i + c_in + e
            uint32_t kbits[2] = {0u, 0u};
            if (DROPOUT) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint4 k4 = keep_row[h][j];
                    kbits[h] = ((k4.x >> c_in) & 0x03030303u) | (((k4.y >> c_in) & 0x03030303u) << 2) |
                               (((k4.z >> c_in) & 0x03030303u) << 4) | (((k4.w >> c_in) & 0x03030303u) << 6);
                }
            }
            const bool piv_tile = SPARSE && j >= nband;
            const int k0 = SPARSE ? (piv_tile ? (j - nband) * BKV : (jb0 + j) * BKV) : j * BKV;
            mbar_wait<false>(&kv_full[stage], phase);
            const uint32_t k_addr = smem_u32(sKV + stage * (K_BYTES + V_BYTES));
            const uint32_t v_addr = k_addr + K_BYTES;
            float s[BKV / 2];
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < HD / 16; ++k)
                wgmma_ss_n128<0, 0>(s, make_smem_desc_sw128(q_addr + k * 32, 0, 1024),
                                    make_smem_desc_sw128(k_addr + k * 32, 0, 1024), k != 0 ? 1u : 0u);
            wgmma_commit();
            // pivot tiles: bit 2i + e of pvis[h] = this thread's gathered key 8i + c_in + e is visible to row h
            uint32_t pvis[2] = {0u, 0u};
            if (piv_tile) {
#pragma unroll
                for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int pj = k0 + 8 * i + c_in + e;
                        const int pp = pj < p.n_piv ? p.piv_pos[(size_t)batch * p.n_piv + pj] : 0x7fffffff;
#pragma unroll
                        for (int h = 0; h < 2; ++h) pvis[h] |= (pp < bs_row[h] ? 1u : 0u) << (2 * i + e);
                    }
            }
            wgmma_wait<0>();
            fence_regs(s);
            float alpha[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                // does this tile need per-element masking for this row?
                const bool full_vis = SPARSE ? (!piv_tile && k0 >= bs_row[h] && k0 + BKV - 1 <= qi[h] && k0 + BKV <= p.sk)
                                             : (k0 + BKV <= p.sk) && ((k0 + BKV <= p.sep_eff) || (k0 + BKV - 1 <= causal_lim[h]));
                float mx = -INFINITY;
#pragma unroll
                for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float& x = s[4 * i + 2 * h + e];
                        const int kj = k0 + 8 * i + c_in + e;
                        float v;
                        if (full_vis) {
                            v = x * p.scale_log2;
                        } else if (piv_tile) {
                            v = ((pvis[h] >> (2 * i + e)) & 1u) ? x * p.scale_log2 + p.piv_bias_log2 : masked_val;
                            if (kj >= p.n_piv) v = -INFINITY;      // beyond the pivot list
                        } else {
                            const bool vis = SPARSE ? (kj >= bs_row[h] && kj <= qi[h])
                                                    : ((kj < p.sep_eff) || (kj <= causal_lim[h]));
                            v = vis ? x * p.scale_log2 : masked_val;
                            if (kj >= p.sk) v = -INFINITY;     // key does not exist
                        }
                        x = v;
                        mx = fmaxf(mx, v);
                    }
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                mx = fmaxf(mx, m[h]);
                alpha[h] = exp2f(m[h] - mx);                // m = -inf on the first tile -> 0
                m[h] = mx;
            }
            uint32_t pk[BKV / 4];                           // bf16 pairs of P in the A-fragment order
            float psum[2] = {0.f, 0.f};
#pragma unroll
            for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float e0 = exp2f(s[4 * i + 2 * h] - m[h]), e1 = exp2f(s[4 * i + 2 * h + 1] - m[h]);
                    uint32_t w = pack_bf16x2(e0, e1);
                    // the row sum uses the bf16-rounded probabilities that the PV MMA will see
                    const __nv_bfloat162 pb = *reinterpret_cast<const __nv_bfloat162*>(&w);
                    psum[h] += __low2float(pb) + __high2float(pb);
                    if (DROPOUT) {   // dropout acts on the normalised probabilities: the row sum stays undropped; the
                                     // 1/(1-p) scale is applied once to the output row at the end
                        const int bit = 8 * (i & 3) + 2 * (i >> 2);
                        w = pack_bf16x2(((kbits[h] >> bit) & 1u) ? e0 : 0.f, ((kbits[h] >> (bit + 1)) & 1u) ? e1 : 0.f);
                    }
                    pk[2 * i + h] = w;
                }
#pragma unroll
            for (int h = 0; h < 2; ++h) l[h] = l[h] * alpha[h] + psum[h];   // this thread's share of the row sum
#pragma unroll
            for (int i = 0; i < HD / 8; ++i) {
                o[4 * i + 0] *= alpha[0]; o[4 * i + 1] *= alpha[0];
                o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
            }
            fence_regs(o);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < BKV / 16; ++kk) {
                uint32_t a[4];
                frag_a(pk, kk, a);
                wgmma_rs_n64<1>(o, a, make_smem_desc_sw128(v_addr + kk * (16 * 128), BKV * 128, 1024), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(o);
            if (lane == 0) mbar_arrive(&kv_empty[stage]);
            if (++stage == KV_STAGES) { stage = 0; phase ^= 1; }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float lt = l[h];
            lt += __shfl_xor_sync(0xffffffffu, lt, 1);
            lt += __shfl_xor_sync(0xffffffffu, lt, 2);
            if (qi[h] < p.sq) {
                const float inv_l = (DROPOUT ? p.drop.scale : 1.0f) / lt;
                __nv_bfloat16* orow = p.out + (size_t)batch * p.bso + (size_t)qi[h] * p.ldo + head * HD;
#pragma unroll
                for (int i = 0; i < HD / 8; ++i)
                    *reinterpret_cast<uint32_t*>(orow + 8 * i + c_in) =
                        pack_bf16x2(o[4 * i + 2 * h] * inv_l, o[4 * i + 2 * h + 1] * inv_l);
                if ((lane & 3) == 0 && p.lse != nullptr)
                    p.lse[((size_t)batch * p.heads + head) * p.sq + qi[h]] = m[h] * 0.6931471805599453f + logf(lt);
            }
        }
    }
}

// Keep decisions of the attention-probability dropout for every (query, key) pair of the visible tiles, generated
// ahead of the attention kernel at full occupancy (inside the attention kernel the same work sits on the softmax
// warps' critical path).  One thread per (query row, key tile): a
// Philox4x32-10 call seeds four 32-step LCG streams, keep iff state >= p * 2^32.  Writes both layouts (AttnParams).
__global__ void __launch_bounds__(128, 4)
attn_dropout_mask_kernel(const AttnParams p) {
    const int qb = blockIdx.x, j = blockIdx.y;
    const int head = blockIdx.z % p.heads, batch = blockIdx.z / p.heads;
    const int q0 = qb * BQ;
    int kmax = q0 + BQ + p.off;
    if (kmax < p.sep_eff) kmax = p.sep_eff;
    if (kmax > p.sk) kmax = p.sk;
    if (j * BKV >= kmax) return;                 // tile never visited by the attention kernels
    const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
    const int qi = q0 + threadIdx.x;
    const uint64_t ctr = (((uint64_t)batch * p.heads + head) * p.sq + qi) * p.nkb_all + j;
    const uint4 r0 = philox4x32_10(p.drop.seed, ctr, p.drop.stream);
    uint32_t rng[4] = {r0.x, r0.y, r0.z, r0.w};
    uint32_t wrow[4], wkey[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        uint32_t bits = 0u, mine = 0u;
#pragma unroll
        for (int t = 0; t < 32; ++t) {
            rng[g] = rng[g] * 1664525u + 1013904223u;
            const bool keep = rng[g] >= p.drop.threshold;
            bits |= (keep ? 1u : 0u) << t;
            const uint32_t bal = __ballot_sync(0xffffffffu, keep);   // key 32g + t over this warp's 32 queries
            if (lane == t) mine = bal;
        }
        wrow[g] = bits;
        wkey[g] = mine;
    }
    const size_t bh = (size_t)batch * p.heads + head;
    const size_t region = (size_t)p.b * p.heads * p.nkb_all * p.nqb_all * (BQ * 4);
    reinterpret_cast<uint4*>(p.drop_mask + region)[(bh * p.nqb_all * BQ + qi) * p.nkb_all + j] =
        make_uint4(wrow[0], wrow[1], wrow[2], wrow[3]);
    uint32_t* dm = p.drop_mask + ((bh * p.nkb_all * BKV + j * BKV + lane) * p.nqb_all + qb) * 4 + wq;
#pragma unroll
    for (int g = 0; g < 4; ++g) dm[(size_t)g * 32 * p.nqb_all * 4] = wkey[g];
}

// [b, s, cols] bf16 view: row stride ld, batch stride bs (elements); box [64 cols x box_rows rows x 1]
int encode_qkv_map(CUtensorMap* m, const void* base, int b, int s, int cols, int64_t ld, int64_t bs, int box_rows) {
    uint64_t dims[3] = {(uint64_t)cols, (uint64_t)s, (uint64_t)b};
    uint64_t str[2] = {(uint64_t)ld * 2, (uint64_t)bs * 2};
    uint32_t box[3] = {64, (uint32_t)box_rows, 1};
    return cvh::encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, str, box, nullptr, cvh::Swizzle::B128);
}

}  // namespace

extern "C" int cv_attn_fwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk,
                           const void* v, int64_t ldv, int64_t bsv, void* out, int64_t ldo, int64_t bso, float* lse,
                           int b, int heads, int head_dim, int sq, int sk, int sep, float dropout_p, uint64_t seed,
                           uint32_t site, uint32_t* drop_mask, void* stream) {
    CV_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "dropout probability must be in [0, 1)");
    CV_REQUIRE(dropout_p == 0.f || drop_mask != nullptr, "attention dropout needs the keep-mask buffer");
    CV_REQUIRE(q && k && v && out, "null pointer");
    CV_REQUIRE(head_dim == HD, "head_dim must be 64 (CogView: hidden / heads = 64)");
    CV_REQUIRE(b > 0 && heads > 0 && sq > 0 && sk >= sq, "need sk >= sq > 0");
    CV_REQUIRE(sep >= 0 && sep <= sq, "sep must be in [0, sq]");
    CV_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && bsq % 8 == 0 && bsk % 8 == 0 &&
                   bsv % 8 == 0 && bso % 8 == 0,
               "strides must be multiples of 8 elements");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    alignas(64) CUtensorMap tmQ, tmK, tmV;
    int rc;
    if ((rc = encode_qkv_map(&tmQ, q, b, sq, heads * HD, ldq, bsq, BQ))) return rc;
    if ((rc = encode_qkv_map(&tmK, k, b, sk, heads * HD, ldk, bsk, BKV))) return rc;
    if ((rc = encode_qkv_map(&tmV, v, b, sk, heads * HD, ldv, bsv, BKV))) return rc;
    AttnParams p;
    p.b = b; p.heads = heads; p.sq = sq; p.sk = sk;
    p.off = sk - sq;
    p.sep_eff = sep > 0 ? sep + (sk - sq) : 0;   // mpu/sparse_transformer.py:486; sep = 0 with memory: see below
    // NB: with sep == 0 the reference still marks the memory columns [0, sk - sq) visible (:486 with sep = 0);
    // they are causally visible anyway (j <= i + off for every i >= 0), so sep_eff = 0 is equivalent.
    p.scale_log2 = (1.0f / sqrtf((float)head_dim)) * LOG2E;
    p.out = static_cast<__nv_bfloat16*>(out);
    p.ldo = ldo; p.bso = bso;
    p.lse = lse;
    {
        const cvh::HostDropout hd = cvh::make_dropout(dropout_p, seed, site);
        p.drop.p = hd.p; p.drop.scale = hd.scale; p.drop.threshold = hd.threshold; p.drop.stream = hd.stream;
        p.drop.seed = hd.seed;
        p.drop_mask = drop_mask;
        p.nkb_all = (sk + BKV - 1) / BKV;
        p.nqb_all = (sq + BQ - 1) / BQ;
        p.keep_q = drop_mask ? drop_mask + (size_t)b * heads * p.nkb_all * p.nqb_all * (BQ * 4) : nullptr;   // region [1]
        p.keep_slots = p.nkb_all;
    }
    p.sp_w = 0; p.sp_times = 0; p.n_piv = 0; p.piv_pos = nullptr; p.piv_bias_log2 = 0.f;
    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        CV_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set = true;
    }
    dim3 grid((sq + BQ - 1) / BQ, heads, b);
    if (dropout_p > 0.f) {
        attn_dropout_mask_kernel<<<dim3(p.nqb_all, p.nkb_all, b * heads), 128, 0, s>>>(p);
        CV_LAUNCH_CHECK();
        attn_fwd_kernel<true, false><<<grid, NUM_THREADS, SMEM_BYTES, s>>>(tmQ, tmK, tmV, tmK, tmV, p);
    }
    else attn_fwd_kernel<false, false><<<grid, NUM_THREADS, SMEM_BYTES, s>>>(tmQ, tmK, tmV, tmK, tmV, p);
    CV_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------------
// sparse training attention (mpu/sparse_transformer.py:675-725): gathered pivots + causal band, one softmax
// ------------------------------------------------------------------------------------------------
namespace {
// gathered pivot keys / values: dst[b, p, 0:h] = K[b, pos[p], :], dst[b, p, h:2h] = V[b, pos[p], :]; pos32 = (int)pos
__global__ void gather_pivots_kernel(const __nv_bfloat16* __restrict__ k, int64_t ldk, int64_t bsk,
                                     const __nv_bfloat16* __restrict__ v, int64_t ldv, int64_t bsv,
                                     const int64_t* __restrict__ pos, __nv_bfloat16* __restrict__ dst,
                                     int* __restrict__ pos32, int b, int n_piv, int h) {
    const int row = blockIdx.x;                 // (batch, pivot)
    const int batch = row / n_piv;
    const int64_t src = pos[row];
    if (threadIdx.x == 0) pos32[row] = (int)src;
    const uint4* ks = reinterpret_cast<const uint4*>(k + (size_t)batch * bsk + (size_t)src * ldk);
    const uint4* vs = reinterpret_cast<const uint4*>(v + (size_t)batch * bsv + (size_t)src * ldv);
    uint4* d = reinterpret_cast<uint4*>(dst + (size_t)row * 2 * h);
    for (int i = threadIdx.x; i < h / 8; i += blockDim.x) {
        d[i] = ks[i];
        d[h / 8 + i] = vs[i];
    }
}

// Keep decisions of the attention-probability dropout of the sparse attention, in the layout of sparse::KeepLayout.
// The keys of query i are virtual: the s sequence positions (band keys), then the n_piv pivot SLOTS (pivot p is its own
// key whatever its position, as column p of the reference's [b, heads, s, n_piv + w*times] probabilities).  One thread
// per (query, virtual key tile) as in attn_dropout_mask_kernel: the Philox4x32-10 call of counter
// ((batch*heads + head)*s + query) * (nkb + npb) + tile seeds four 32-step LCG streams, keep iff state >= p * 2^32.
// A tile is written to the forward region and/or to the backward region of its pass when that kernel visits it.
__global__ void __launch_bounds__(128, 4)
attn_sparse_dropout_mask_kernel(const DropoutArgs drop, uint32_t* __restrict__ mask, const sparse::KeepLayout L,
                                int heads, int s, int w, int times) {
    const int qb = blockIdx.x, vb = blockIdx.y;
    const int head = blockIdx.z % heads, batch = blockIdx.z / heads;
    int fslot = -1, bslot = -1;            // entry of this tile in the forward / backward walk, -1: not visited
    if (vb < L.nkb) {
        const int jb0 = sparse::fwd_band_first(qb, w, times);
        if (vb >= jb0 && vb < jb0 + sparse::fwd_band_count(qb, s, w, times)) fslot = vb - jb0;
        if (qb >= vb && qb <= sparse::bwd_band_last(vb, L.nqb, w, times)) bslot = qb - vb;
    } else {
        if (sparse::fwd_sees_pivots(qb, s, w, times)) fslot = sparse::fwd_band_count(qb, s, w, times) + vb - L.nkb;
        if (L.np > 0 && qb >= sparse::piv_first(w, times)) bslot = qb - sparse::piv_first(w, times);
    }
    if (fslot < 0 && bslot < 0) return;
    const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
    const int qi = qb * BQ + threadIdx.x;
    const size_t bh = (size_t)batch * heads + head;
    const uint64_t ctr = ((uint64_t)bh * s + qi) * (uint64_t)(L.nkb + L.npb) + vb;
    const uint4 r0 = philox4x32_10(drop.seed, ctr, drop.stream);
    uint32_t rng[4] = {r0.x, r0.y, r0.z, r0.w};
    uint32_t wrow[4], wkey[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        uint32_t bits = 0u, mine = 0u;
#pragma unroll
        for (int t = 0; t < 32; ++t) {
            rng[g] = rng[g] * 1664525u + 1013904223u;
            const bool keep = rng[g] >= drop.threshold;
            bits |= (keep ? 1u : 0u) << t;
            const uint32_t bal = __ballot_sync(0xffffffffu, keep);   // key 32g + t over this warp's 32 queries
            if (lane == t) mine = bal;
        }
        wrow[g] = bits;
        wkey[g] = mine;
    }
    if (fslot >= 0)
        reinterpret_cast<uint4*>(mask)[(bh * L.nqb * BQ + qi) * (L.tb + L.npb) + fslot] =
            make_uint4(wrow[0], wrow[1], wrow[2], wrow[3]);
    if (bslot >= 0) {
        const bool band = vb < L.nkb;
        const int slots = band ? L.tq : L.np;
        const size_t rows = (size_t)(band ? L.nkb : L.npb) * BKV;        // key rows per (batch, head)
        const int key0 = (band ? vb : vb - L.nkb) * BKV;
        uint32_t* dm = mask + L.fwd_words + (band ? 0 : L.band_words) +
                       ((bh * rows + key0 + lane) * slots + bslot) * 4 + wq;
#pragma unroll
        for (int g = 0; g < 4; ++g) dm[(size_t)g * 32 * slots * 4] = wkey[g];
    }
}
}  // namespace

extern "C" int64_t cv_attn_sparse_workspace_bytes(int b, int heads, int head_dim, int n_piv) {
    const int64_t h = (int64_t)heads * head_dim;
    return ((int64_t)b * n_piv * 2 * h * 2 + 255) / 256 * 256 + (int64_t)b * n_piv * 4;
}

extern "C" int64_t cv_attn_sparse_drop_mask_words(int b, int heads, int s, int n_piv, int query_window,
                                                  int key_window_times) {
    CV_REQUIRE(b > 0 && heads > 0 && s > 0 && n_piv > 0 && n_piv <= s, "bad sizes");
    CV_REQUIRE(query_window > 0 && key_window_times > 0 && s % query_window == 0,
               "the sequence length must be a multiple of query_window");
    const sparse::KeepLayout L = sparse::keep_layout(b, heads, s, n_piv, query_window, key_window_times);
    return L.fwd_words + L.band_words + L.piv_words;
}

namespace {
int attn_sparse_fwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk, const void* v,
                    int64_t ldv, int64_t bsv, const int64_t* pivot_idx, void* out, int64_t ldo, int64_t bso, float* lse,
                    void* workspace, int b, int heads, int head_dim, int s, int n_piv, int query_window,
                    int key_window_times, float dropout_p, uint64_t seed, uint32_t site, uint32_t* drop_mask,
                    cudaStream_t st) {
    CV_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "dropout probability must be in [0, 1)");
    CV_REQUIRE(dropout_p == 0.f || drop_mask != nullptr, "attention dropout needs the keep-mask buffer");
    CV_REQUIRE(q && k && v && pivot_idx && out && workspace, "null pointer");
    CV_REQUIRE(head_dim == HD, "head_dim must be 64 (CogView: hidden / heads = 64)");
    CV_REQUIRE(b > 0 && heads > 0 && s > 0 && n_piv > 0 && n_piv <= s, "bad sizes");
    CV_REQUIRE(query_window > 0 && key_window_times > 0 && s % query_window == 0,
               "the sequence length must be a multiple of query_window (mpu/sparse_transformer.py:703,713)");
    CV_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && bsq % 8 == 0 && bsk % 8 == 0 &&
                   bsv % 8 == 0 && bso % 8 == 0,
               "strides must be multiples of 8 elements");
    const int h = heads * HD;
    __nv_bfloat16* pkv = static_cast<__nv_bfloat16*>(workspace);
    int* pos32 = reinterpret_cast<int*>(static_cast<char*>(workspace) + ((size_t)b * n_piv * 2 * h * 2 + 255) / 256 * 256);
    gather_pivots_kernel<<<b * n_piv, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(k), ldk, bsk,
                                                   static_cast<const __nv_bfloat16*>(v), ldv, bsv, pivot_idx, pkv, pos32,
                                                   b, n_piv, h);
    CV_LAUNCH_CHECK();
    alignas(64) CUtensorMap tmQ, tmK, tmV, tmPK, tmPV;
    int rc;
    if ((rc = encode_qkv_map(&tmQ, q, b, s, h, ldq, bsq, BQ))) return rc;
    if ((rc = encode_qkv_map(&tmK, k, b, s, h, ldk, bsk, BKV))) return rc;
    if ((rc = encode_qkv_map(&tmV, v, b, s, h, ldv, bsv, BKV))) return rc;
    if ((rc = encode_qkv_map(&tmPK, pkv, b, n_piv, h, 2 * (int64_t)h, (int64_t)n_piv * 2 * h, BKV))) return rc;
    if ((rc = encode_qkv_map(&tmPV, pkv + h, b, n_piv, h, 2 * (int64_t)h, (int64_t)n_piv * 2 * h, BKV))) return rc;
    AttnParams p;
    p.b = b; p.heads = heads; p.sq = s; p.sk = s;
    p.off = 0; p.sep_eff = 0;
    p.scale_log2 = (1.0f / sqrtf((float)head_dim)) * LOG2E;
    p.out = static_cast<__nv_bfloat16*>(out);
    p.ldo = ldo; p.bso = bso; p.lse = lse;
    const cvh::HostDropout hd = cvh::make_dropout(dropout_p, seed, site);
    p.drop.p = hd.p; p.drop.scale = hd.scale; p.drop.threshold = hd.threshold; p.drop.stream = hd.stream;
    p.drop.seed = hd.seed;
    p.drop_mask = drop_mask;
    p.nkb_all = (s + BKV - 1) / BKV;
    p.nqb_all = (s + BQ - 1) / BQ;
    p.sp_w = query_window; p.sp_times = key_window_times; p.n_piv = n_piv; p.piv_pos = pos32;
    p.piv_bias_log2 = logf((float)(s / n_piv)) * LOG2E;           // integer division as in :697
    const sparse::KeepLayout L = sparse::keep_layout(b, heads, s, n_piv, query_window, key_window_times);
    p.keep_q = drop_mask;                                         // the forward region comes first
    p.keep_slots = L.tb + L.npb;
    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        CV_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set = true;
    }
    dim3 grid((s + BQ - 1) / BQ, heads, b);
    if (dropout_p > 0.f) {
        attn_sparse_dropout_mask_kernel<<<dim3(L.nqb, L.nkb + L.npb, b * heads), 128, 0, st>>>(
            p.drop, drop_mask, L, heads, s, query_window, key_window_times);
        CV_LAUNCH_CHECK();
        attn_fwd_kernel<true, true><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(tmQ, tmK, tmV, tmPK, tmPV, p);
    } else {
        attn_fwd_kernel<false, true><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(tmQ, tmK, tmV, tmPK, tmPV, p);
    }
    CV_LAUNCH_CHECK();
    return 0;
}
}  // namespace

extern "C" int cv_attn_sparse_fwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk,
                                  const void* v, int64_t ldv, int64_t bsv, const int64_t* pivot_idx, void* out,
                                  int64_t ldo, int64_t bso, float* lse, void* workspace, int b, int heads,
                                  int head_dim, int s, int n_piv, int query_window, int key_window_times,
                                  void* stream) {
    return attn_sparse_fwd(q, ldq, bsq, k, ldk, bsk, v, ldv, bsv, pivot_idx, out, ldo, bso, lse, workspace, b, heads,
                           head_dim, s, n_piv, query_window, key_window_times, 0.f, 0, 0, nullptr,
                           static_cast<cudaStream_t>(stream));
}

extern "C" int cv_attn_sparse_fwd_dropout(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk,
                                          int64_t bsk, const void* v, int64_t ldv, int64_t bsv, const int64_t* pivot_idx,
                                          void* out, int64_t ldo, int64_t bso, float* lse, void* workspace, int b,
                                          int heads, int head_dim, int s, int n_piv, int query_window,
                                          int key_window_times, float dropout_p, uint64_t seed, uint32_t site,
                                          uint32_t* drop_mask, void* stream) {
    return attn_sparse_fwd(q, ldq, bsq, k, ldk, bsk, v, ldv, bsv, pivot_idx, out, ldo, bso, lse, workspace, b, heads,
                           head_dim, s, n_piv, query_window, key_window_times, dropout_p, seed, site, drop_mask,
                           static_cast<cudaStream_t>(stream));
}
