// cv_attn_bwd: backward of the fused dense attention (autograd of standard_attention,
// /root/reference/mpu/sparse_transformer.py:652-673, which the reference gets from torch autograd over
// materialised [b, np, s, s] tensors).  Recomputes P from Q, K and the saved log-sum-exp; nothing of
// size [s, s] reaches HBM.
//
//   P = exp(S - lse),  S = scale * Q K^T (masked entries: -10000, gradient 0)
//   dV = P^T dO        dP = dO V^T        dS = P o (dP - D),  D = rowsum(dO o O)
//   dQ = scale * dS K  dK = scale * dS^T Q
//
// One CTA per (128-key block, head, batch) loops over the query blocks that can see it: a TMA producer warpgroup
// and two wgmma warpgroups that own 64 key rows each.  All five products run on wgmma with fp32 accumulators in
// registers; the shared-memory operands are used in place from 128B-swizzled TMA tiles, in K-major or MN-major
// form as the product needs (the same Q / dO / K tiles serve both):
//   S^T  = K Q^T      (A = K   K-major, B = Q  K-major)   [keys x queries]
//   dP^T = V dO^T     (A = V   K-major, B = dO K-major)
//   dV  += P^T dO     (A = P^T from registers,  B = dO MN-major)
//   dK  += dS^T Q     (A = dS^T from registers, B = Q  MN-major)
//   dQ_i = dS K       (A = dS^T of both warpgroups, written to smem and read MN-major, B = K MN-major)
// dV / dK stay in registers for the whole loop; dQ tiles are reduced into an fp32 buffer with vector red.add.
#include "attention_sparse.cuh"
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

constexpr int BLK = 128;
constexpr int HD = 64;
constexpr int TILE_BYTES = BLK * HD * 2;      // 16 KB: one [128 x 64] bf16 tile
constexpr int PT_BYTES = BLK * BLK * 2;       // 32 KB: [128 keys x 128 queries] bf16
constexpr int QDO_STAGES = 2;
constexpr int SMEM_BYTES = 2 * TILE_BYTES /*K,V*/ + QDO_STAGES * 2 * TILE_BYTES /*Q,dO*/ + 2 * PT_BYTES /*dS^T x 2*/ +
                           2 * 2 * 3 * BLK * 4 /*per warpgroup, 2 buffers: lse2, D, band start*/ + 1024 + 256;
enum { MODE_DENSE = 0, MODE_BAND = 1, MODE_PIVOT = 2 };
constexpr int NUM_THREADS = 384;     // TMA warpgroup, two wgmma warpgroups (64 key rows each)
constexpr float LOG2E = 1.4426950408889634f;

struct BwdParams {
    int b, heads, s;
    int sep_eff;
    float scale, scale_log2;
    const float* lse;    // [b, heads, s]
    const float* delta;  // [b, heads, s]
    float* dq_acc;       // [b, s, heads*HD] fp32, zero-initialised
    __nv_bfloat16* dqkv; // [b, s, 3*heads*HD]
    const uint32_t* drop_mask;  // keep bits written by the forward, key-major ([b, heads, keep_rows, keep_slots, 4]: the 128
                                // query bits of (key, query tile) are one 16-byte load for the thread that owns the key) or
                                // null.  Dense: keep_rows = nqb*128, slot = query block; sparse: the band / pivot region of
                                // sparse::KeepLayout, slot = local query-tile counter t
    int keep_rows, keep_slots;
    float drop_scale;           // 1 / (1 - p)
    // sparse training attention (mpu/sparse_transformer.py:675-725), two launches that share lse / delta / dq_acc:
    //   MODE_BAND : keys = the sequence, key j visible to query i iff band_start(i) <= j <= i
    //   MODE_PIVOT: keys = the gathered pivots (sk = n_piv rows), pivot visible iff piv_pos < band_start(i),
    //               scores carry + log(s / n_piv); dK / dV rows go to the gathered scratch (kv_rows = n_piv)
    int sk, kv_rows, sp_w, sp_times;
    const int* piv_pos;         // [b, sk]
    float piv_bias_log2;
};

using sparse::band_start;

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO, const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sK = smem;
    uint8_t* sV = sK + TILE_BYTES;
    uint8_t* sQDO = sV + TILE_BYTES;                               // stage s: Q then dO
    uint8_t* sDST = sQDO + QDO_STAGES * 2 * TILE_BYTES;            // [2 buffers] dS^T [128 keys x 128 queries]
    float* sStat = reinterpret_cast<float*>(sDST + 2 * PT_BYTES);  // [warpgroup][buffer][lse2 | D | band] x 128
    uint64_t* bars = reinterpret_cast<uint64_t*>(sStat + 2 * 2 * 3 * BLK);
    uint64_t* kv_full = bars;                  // 1
    uint64_t* qdo_full = bars + 1;             // [2]
    uint64_t* qdo_empty = qdo_full + QDO_STAGES;   // [2]: one arrive per consumer warp

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int kb = blockIdx.x, head = blockIdx.y, batch = blockIdx.z;
    const int k0 = kb * BLK;
    const int nqb = (p.s + BLK - 1) / BLK;
    // query blocks that can see a key of this block
    int i_start = (k0 < p.sep_eff) ? 0 : kb, i_end = nqb - 1;
    if (MODE == MODE_BAND) {          // queries i with band_start(i) <= j <= i
        i_start = kb;
        i_end = sparse::bwd_band_last(kb, nqb, p.sp_w, p.sp_times);
    } else if (MODE == MODE_PIVOT) {  // band_start(i) > 0  <=>  i >= sp_times * sp_w   (the host checks this is < s)
        i_start = sparse::piv_first(p.sp_w, p.sp_times);
    }
    const int ntiles = i_end - i_start + 1;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO);
        mbar_init(kv_full, 1);
        for (int i = 0; i < QDO_STAGES; ++i) { mbar_init(&qdo_full[i], 1); mbar_init(&qdo_empty[i], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tid == 0) {
            mbar_expect_tx(kv_full, 2 * TILE_BYTES);
            tma_load_3d(sK, &tmK, kv_full, head * HD, k0, batch);
            tma_load_3d(sV, &tmV, kv_full, head * HD, k0, batch);
            int stage = 0; uint32_t phase = 0;
            for (int t = 0; t < ntiles; ++t) {
                const int q0 = (i_start + t) * BLK;
                mbar_wait<false>(&qdo_empty[stage], phase ^ 1);
                uint8_t* sQ = sQDO + stage * 2 * TILE_BYTES;
                mbar_expect_tx(&qdo_full[stage], 2 * TILE_BYTES);
                tma_load_3d(sQ, &tmQ, &qdo_full[stage], head * HD, q0, batch);
                tma_load_3d(sQ + TILE_BYTES, &tmDO, &qdo_full[stage], head * HD, q0, batch);
                if (++stage == QDO_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // Fragment layout (common.cuh): this thread holds key rows r_loc, r_loc + 8 of the block and, of every
        // 8-query group of a tile, the two queries c_in, c_in + 1.  For dQ (rows = queries) the same positions index
        // queries 64 half + ... and head dims.
        setmaxnreg_inc<232>();
        const int half = wg - 1, warp = tid >> 5, lane = tid & 31;
        const int r_loc = 64 * half + 16 * warp + (lane >> 2);
        const int c_in = 2 * (lane & 3);
        const float masked_val = -10000.0f * LOG2E;
        int kj[2], my_pos[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            kj[h] = k0 + r_loc + 8 * h;
            my_pos[h] = (MODE == MODE_PIVOT) ? (kj[h] < p.sk ? p.piv_pos[(size_t)batch * p.sk + kj[h]] : 0x7fffffff) : 0;
        }
        const size_t stat_base = ((size_t)batch * p.heads + head) * p.s;
        const size_t keep_base = ((size_t)batch * p.heads + head) * (size_t)p.keep_rows;   // key rows are padded to blocks
        const int keep_slot0 = MODE == MODE_DENSE ? i_start : 0;
        const uint32_t k_addr = smem_u32(sK), v_addr = smem_u32(sV);
        const uint32_t kh_addr = k_addr + half * (64 * 128), vh_addr = v_addr + half * (64 * 128);
        float dv[HD / 2], dk[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
        mbar_wait<false>(kv_full, 0);
        int stage = 0; uint32_t phase = 0;
        for (int t = 0; t < ntiles; ++t) {
            const int q0 = (i_start + t) * BLK;
            const int buf = t & 1;
            // per-query statistics of this tile (lse in the log2 domain, delta, band start) -> this warpgroup's buffer
            float* st = sStat + (half * 2 + buf) * 3 * BLK;
            {
                const int qn = q0 + tid;
                st[tid] = (qn < p.s) ? p.lse[stat_base + qn] * LOG2E : 0.f;
                st[BLK + tid] = (qn < p.s) ? p.delta[stat_base + qn] : 0.f;
                if (MODE != MODE_DENSE) reinterpret_cast<int*>(st)[2 * BLK + tid] = band_start(qn, p.sp_w, p.sp_times);
            }
            uint4 kw[2] = {make_uint4(0u, 0u, 0u, 0u), make_uint4(0u, 0u, 0u, 0u)};
            const bool use_drop = p.drop_mask != nullptr;
            if (use_drop) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    kw[h] = *reinterpret_cast<const uint4*>(p.drop_mask +
                                                            ((keep_base + kj[h]) * (size_t)p.keep_slots + keep_slot0 + t) * 4);
            }
            named_bar_sync(1 + half, 128);
            mbar_wait<false>(&qdo_full[stage], phase);
            const uint32_t q_addr = smem_u32(sQDO + stage * 2 * TILE_BYTES);
            const uint32_t do_addr = q_addr + TILE_BYTES;
            float sacc[BLK / 2], dpacc[BLK / 2];
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < HD / 16; ++k)
                wgmma_ss_n128<0, 0>(sacc, make_smem_desc_sw128(kh_addr + k * 32, 0, 1024),
                                    make_smem_desc_sw128(q_addr + k * 32, 0, 1024), k != 0 ? 1u : 0u);
            wgmma_commit();
#pragma unroll
            for (int k = 0; k < HD / 16; ++k)
                wgmma_ss_n128<0, 0>(dpacc, make_smem_desc_sw128(vh_addr + k * 32, 0, 1024),
                                    make_smem_desc_sw128(do_addr + k * 32, 0, 1024), k != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(sacc);
            fence_regs(dpacc);
            bool full_vis = (q0 + BLK <= p.s) && (k0 + BLK <= p.s) &&
                            ((k0 + BLK <= p.sep_eff) || (k0 + BLK - 1 <= q0));
            if (MODE == MODE_BAND)      // every key of the block inside the band of every query of the tile
                full_vis = (q0 + BLK <= p.s) && (k0 + BLK - 1 <= q0) &&
                           (k0 >= band_start(q0 + BLK - 1, p.sp_w, p.sp_times));
            if (MODE == MODE_PIVOT) full_vis = false;
            const float* lse2 = st;
            const float* dlt = st + BLK;
            const int* bnd = reinterpret_cast<const int*>(st) + 2 * BLK;
            uint32_t ppk[BLK / 4], dspk[BLK / 4];      // bf16 pairs of P^T (dropped) and dS^T, A-fragment order
#pragma unroll
            for (int i = 0; i < BLK / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float pv[2], dsv[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * i + c_in + e;
                        const int qi = q0 + col;
                        float s2 = sacc[4 * i + 2 * h + e] * p.scale_log2;
                        float pr;
                        if (full_vis) {
                            pr = exp2f(s2 - lse2[col]);
                        } else if (MODE == MODE_PIVOT) {
                            const bool vis = my_pos[h] < bnd[col];
                            s2 = vis ? s2 + p.piv_bias_log2 : masked_val;
                            pr = (kj[h] < p.sk && qi < p.s) ? exp2f(s2 - lse2[col]) : 0.f;
                        } else {
                            const bool vis = (MODE == MODE_BAND) ? (kj[h] >= bnd[col] && kj[h] <= qi)
                                                                 : ((kj[h] < p.sep_eff) || (kj[h] <= qi));
                            if (!vis) s2 = masked_val;
                            pr = (kj[h] < p.s && qi < p.s) ? exp2f(s2 - lse2[col]) : 0.f;
                        }
                        float dp = dpacc[4 * i + 2 * h + e];
                        float pdrop = pr;
                        if (use_drop) {   // dP flows back through the keep mask; dV sees the dropped probabilities
                            const uint4 k4 = kw[h];
                            const int wi = col >> 5;
                            const uint32_t word = wi == 0 ? k4.x : (wi == 1 ? k4.y : (wi == 2 ? k4.z : k4.w));
                            const bool keep = (word >> (col & 31)) & 1u;
                            dp = keep ? dp * p.drop_scale : 0.f;
                            pdrop = keep ? pr * p.drop_scale : 0.f;
                        }
                        pv[e] = pdrop;
                        dsv[e] = pr * (dp - dlt[col]) * p.scale;
                    }
                    ppk[2 * i + h] = pack_bf16x2(pv[0], pv[1]);
                    dspk[2 * i + h] = pack_bf16x2(dsv[0], dsv[1]);
                }
            // dS^T -> shared memory (128B-swizzled, two 64-query sub-tiles) for the dQ product of both warpgroups
            uint8_t* dbuf = sDST + buf * PT_BYTES;
#pragma unroll
            for (int i = 0; i < BLK / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = r_loc + 8 * h;
                    const int sub = i >> 3, chunk = i & 7;
                    *reinterpret_cast<uint32_t*>(dbuf + sub * (BLK * 128) + row * 128 + ((chunk ^ (row & 7)) << 4) +
                                                 2 * c_in) = dspk[2 * i + h];
                }
            fence_proxy_async_smem();
            // dV += P^T dO,  dK += dS^T Q   (reduction over the 128 queries of this tile)
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLK / 16; ++k) {
                uint32_t a[4];
                frag_a(ppk, k, a);
                wgmma_rs_n64<1>(dv, a, make_smem_desc_sw128(do_addr + k * 2048, BLK * 128, 1024), 1u);
                frag_a(dspk, k, a);
                wgmma_rs_n64<1>(dk, a, make_smem_desc_sw128(q_addr + k * 2048, BLK * 128, 1024), 1u);
            }
            wgmma_commit();
            named_bar_sync(3, 256);                    // both halves of dS^T written
            // dQ rows 64 half .. +63 of this query tile = dS K  (reduction over the 128 keys of this block)
            float dq[HD / 2];
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLK / 16; ++k)
                wgmma_ss_n64<1, 1>(dq, make_smem_desc_sw128(smem_u32(dbuf) + half * (BLK * 128) + k * 2048, BLK * 128, 1024),
                                   make_smem_desc_sw128(k_addr + k * 2048, BLK * 128, 1024), k != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(dv);
            fence_regs(dk);
            fence_regs(dq);
            if (lane == 0) mbar_arrive(&qdo_empty[stage]);
            if (++stage == QDO_STAGES) { stage = 0; phase ^= 1; }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int qi = q0 + r_loc + 8 * h;     // dQ tile rows are queries
                if (qi < p.s) {
                    float* dst = p.dq_acc + ((size_t)batch * p.s + qi) * (p.heads * HD) + head * HD;
#pragma unroll
                    for (int i = 0; i < HD / 8; ++i) red_add_v2(dst + 8 * i + c_in, dq[4 * i + 2 * h], dq[4 * i + 2 * h + 1]);
                }
            }
        }
        // dK / dV of this key block
        const int H3 = 3 * p.heads * HD;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (kj[h] >= p.kv_rows) continue;
            __nv_bfloat16* base = p.dqkv + ((size_t)batch * p.kv_rows + kj[h]) * H3 + head * HD;
#pragma unroll
            for (int i = 0; i < HD / 8; ++i) {
                *reinterpret_cast<uint32_t*>(base + p.heads * HD + 8 * i + c_in) =
                    pack_bf16x2(dk[4 * i + 2 * h], dk[4 * i + 2 * h + 1]);
                *reinterpret_cast<uint32_t*>(base + 2 * p.heads * HD + 8 * i + c_in) =
                    pack_bf16x2(dv[4 * i + 2 * h], dv[4 * i + 2 * h + 1]);
            }
        }
    }
}

// delta[b, head, q] = sum_d dO[b, q, head, d] * O[b, q, head, d]
__global__ void attn_bwd_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o,
                                      float* __restrict__ delta, int b, int heads, int s) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;   // (batch, q, head), head fastest
    if (idx >= b * s * heads) return;
    const int head = idx % heads;
    const int tok = idx / heads;
    const uint4* po = reinterpret_cast<const uint4*>(o + (size_t)tok * heads * HD + head * HD);
    const uint4* pd = reinterpret_cast<const uint4*>(d_o + (size_t)tok * heads * HD + head * HD);
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
        uint4 a = po[i], c = pd[i];
        const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a);
        const __nv_bfloat162* pc = reinterpret_cast<const __nv_bfloat162*>(&c);
#pragma unroll
        for (int t = 0; t < 4; ++t)
            acc += __low2float(pa[t]) * __low2float(pc[t]) + __high2float(pa[t]) * __high2float(pc[t]);
    }
    const int bi = tok / s, qi = tok % s;
    delta[((size_t)bi * heads + head) * s + qi] = acc;
}

// dqkv[:, 0:h] = bf16(dq_acc)
__global__ void attn_bwd_dq_store_kernel(const float* __restrict__ dq, __nv_bfloat16* __restrict__ dqkv, size_t rows,
                                         int h) {
    const size_t n4 = rows * (size_t)(h / 4);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / (h / 4);
        const int c = (int)(i % (h / 4)) * 4;
        float4 v = *reinterpret_cast<const float4*>(dq + r * h + c);
        uint2 u;
        u.x = pack_bf16x2(v.x, v.y);
        u.y = pack_bf16x2(v.z, v.w);
        *reinterpret_cast<uint2*>(dqkv + r * 3 * h + c) = u;
    }
}

int encode_map3(CUtensorMap* m, const void* base, int b, int s, int cols, int64_t ld, int64_t bs) {
    uint64_t dims[3] = {(uint64_t)cols, (uint64_t)s, (uint64_t)b};
    uint64_t str[2] = {(uint64_t)ld * 2, (uint64_t)bs * 2};
    uint32_t box[3] = {64, BLK, 1};
    return cvh::encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, str, box, nullptr, cvh::Swizzle::B128);
}

}  // namespace

extern "C" int64_t cv_attn_bwd_workspace_bytes(int b, int heads, int head_dim, int s) {
    return (int64_t)b * s * heads * head_dim * 4 /*dq fp32*/ + (int64_t)b * heads * s * 4 /*delta*/;
}

extern "C" int cv_attn_bwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk,
                           const void* v, int64_t ldv, int64_t bsv, const void* out, const void* d_out,
                           const float* lse, void* dqkv, void* workspace, int b, int heads, int head_dim, int s,
                           int sep, float dropout_p, const uint32_t* drop_mask, void* stream) {
    CV_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "dropout probability must be in [0, 1)");
    CV_REQUIRE(dropout_p == 0.f || drop_mask != nullptr, "attention dropout needs the keep mask saved by the forward");
    CV_REQUIRE(q && k && v && out && d_out && lse && dqkv && workspace, "null pointer");
    CV_REQUIRE(head_dim == HD, "head_dim must be 64");
    CV_REQUIRE(b > 0 && heads > 0 && s > 0 && sep >= 0 && sep <= s, "bad sizes");
    CV_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && bsq % 8 == 0 && bsk % 8 == 0 && bsv % 8 == 0,
               "strides must be multiples of 8 elements");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int h = heads * HD;
    float* dq_acc = static_cast<float*>(workspace);
    float* delta = dq_acc + (size_t)b * s * h;
    CV_CUDA(cudaMemsetAsync(dq_acc, 0, (size_t)b * s * h * sizeof(float), st));
    {
        const int n = b * s * heads;
        attn_bwd_delta_kernel<<<(n + 255) / 256, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(out),
                                                              static_cast<const __nv_bfloat16*>(d_out), delta, b,
                                                              heads, s);
        CV_LAUNCH_CHECK();
    }
    alignas(64) CUtensorMap tmQ, tmK, tmV, tmDO;
    int rc;
    if ((rc = encode_map3(&tmQ, q, b, s, h, ldq, bsq))) return rc;
    if ((rc = encode_map3(&tmK, k, b, s, h, ldk, bsk))) return rc;
    if ((rc = encode_map3(&tmV, v, b, s, h, ldv, bsv))) return rc;
    if ((rc = encode_map3(&tmDO, d_out, b, s, h, h, (int64_t)s * h))) return rc;
    BwdParams p;
    p.b = b; p.heads = heads; p.s = s;
    p.sep_eff = sep;
    p.scale = 1.0f / sqrtf((float)head_dim);
    p.scale_log2 = p.scale * LOG2E;
    p.lse = lse; p.delta = delta; p.dq_acc = dq_acc;
    p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
    p.drop_mask = dropout_p > 0.f ? drop_mask : nullptr;
    p.drop_scale = dropout_p > 0.f ? 1.0f / (1.0f - dropout_p) : 1.0f;
    p.keep_rows = ((s + BLK - 1) / BLK) * BLK;
    p.keep_slots = (s + BLK - 1) / BLK;
    p.sk = s; p.kv_rows = s; p.sp_w = 1; p.sp_times = 1; p.piv_pos = nullptr; p.piv_bias_log2 = 0.f;
    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<MODE_DENSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set = true;
    }
    dim3 grid((s + BLK - 1) / BLK, heads, b);
    attn_bwd_kernel<MODE_DENSE><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(tmQ, tmK, tmV, tmDO, p);
    CV_LAUNCH_CHECK();
    {
        const size_t rows = (size_t)b * s;
        const size_t n4 = rows * (h / 4);
        size_t blocks = (n4 + 255) / 256;
        size_t cap = (size_t)cvh::num_sms() * 8;
        attn_bwd_dq_store_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(
            dq_acc, static_cast<__nv_bfloat16*>(dqkv), rows, h);
        CV_LAUNCH_CHECK();
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// backward of the sparse training attention: band pass + gathered-pivot pass with the JOINT lse and
// delta = rowsum(dO o O); the pivot pass' dK / dV are scattered back to the pivot positions
// (oracle/sparse_decomposition.py: sparse_attention_two_pass_backward)
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void gather_pivots_bwd_kernel(const __nv_bfloat16* __restrict__ k, int64_t ldk, int64_t bsk,
                                         const __nv_bfloat16* __restrict__ v, int64_t ldv, int64_t bsv,
                                         const int64_t* __restrict__ pos, __nv_bfloat16* __restrict__ dst,
                                         int* __restrict__ pos32, int n_piv, int h) {
    const int row = blockIdx.x;
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

// dqkv[b, pos[p], h:3h] += dpiv[b, p, h:3h]   (pivot positions of one sequence are distinct: no atomics)
__global__ void scatter_pivot_grads_kernel(const __nv_bfloat16* __restrict__ dpiv, const int* __restrict__ pos32,
                                           __nv_bfloat16* __restrict__ dqkv, int n_piv, int s, int h) {
    const int row = blockIdx.x;
    const int batch = row / n_piv;
    const __nv_bfloat162* src = reinterpret_cast<const __nv_bfloat162*>(dpiv + (size_t)row * 3 * h + h);
    __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(dqkv + ((size_t)batch * s + pos32[row]) * 3 * h + h);
    for (int i = threadIdx.x; i < h; i += blockDim.x) {          // 2h bf16 = h pairs
        const float2 a = __bfloat1622float2(dst[i]), c = __bfloat1622float2(src[i]);
        dst[i] = __floats2bfloat162_rn(a.x + c.x, a.y + c.y);
    }
}
inline size_t al256b(size_t x) { return (x + 255) / 256 * 256; }
}  // namespace

extern "C" int64_t cv_attn_sparse_bwd_workspace_bytes(int b, int heads, int head_dim, int s, int n_piv) {
    const size_t h = (size_t)heads * head_dim;
    return (int64_t)(al256b((size_t)b * s * h * 4) + al256b((size_t)b * heads * s * 4) + al256b((size_t)b * n_piv * 2 * h * 2) +
                     al256b((size_t)b * n_piv * 3 * h * 2) + al256b((size_t)b * n_piv * 4));
}

extern "C" int cv_attn_sparse_bwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk,
                                  const void* v, int64_t ldv, int64_t bsv, const int64_t* pivot_idx, const void* out,
                                  const void* d_out, const float* lse, void* dqkv, void* workspace, int b, int heads,
                                  int head_dim, int s, int n_piv, int query_window, int key_window_times,
                                  float dropout_p, const uint32_t* drop_mask, void* stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    CV_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "dropout probability must be in [0, 1)");
    CV_REQUIRE(dropout_p == 0.f || drop_mask != nullptr, "attention dropout needs the keep mask saved by the forward");
    CV_REQUIRE(q && k && v && pivot_idx && out && d_out && lse && dqkv && workspace, "null pointer");
    CV_REQUIRE(head_dim == HD, "head_dim must be 64");
    CV_REQUIRE(b > 0 && heads > 0 && s > 0 && n_piv > 0 && n_piv <= s, "bad sizes");
    CV_REQUIRE(query_window > 0 && key_window_times > 0 && s % query_window == 0,
               "the sequence length must be a multiple of query_window");
    CV_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && bsq % 8 == 0 && bsk % 8 == 0 && bsv % 8 == 0,
               "strides must be multiples of 8 elements");
    const int h = heads * HD;
    char* ws = static_cast<char*>(workspace);
    float* dq_acc = reinterpret_cast<float*>(ws);
    ws += al256b((size_t)b * s * h * 4);
    float* delta = reinterpret_cast<float*>(ws);
    ws += al256b((size_t)b * heads * s * 4);
    __nv_bfloat16* pkv = reinterpret_cast<__nv_bfloat16*>(ws);
    ws += al256b((size_t)b * n_piv * 2 * h * 2);
    __nv_bfloat16* dpiv = reinterpret_cast<__nv_bfloat16*>(ws);
    ws += al256b((size_t)b * n_piv * 3 * h * 2);
    int* pos32 = reinterpret_cast<int*>(ws);
    CV_CUDA(cudaMemsetAsync(dq_acc, 0, (size_t)b * s * h * sizeof(float), st));
    {
        const int n = b * s * heads;
        attn_bwd_delta_kernel<<<(n + 255) / 256, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(out),
                                                              static_cast<const __nv_bfloat16*>(d_out), delta, b,
                                                              heads, s);
        CV_LAUNCH_CHECK();
    }
    gather_pivots_bwd_kernel<<<b * n_piv, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(k), ldk, bsk,
                                                       static_cast<const __nv_bfloat16*>(v), ldv, bsv, pivot_idx, pkv,
                                                       pos32, n_piv, h);
    CV_LAUNCH_CHECK();
    alignas(64) CUtensorMap tmQ, tmK, tmV, tmDO, tmPK, tmPV;
    int rc;
    if ((rc = encode_map3(&tmQ, q, b, s, h, ldq, bsq))) return rc;
    if ((rc = encode_map3(&tmK, k, b, s, h, ldk, bsk))) return rc;
    if ((rc = encode_map3(&tmV, v, b, s, h, ldv, bsv))) return rc;
    if ((rc = encode_map3(&tmDO, d_out, b, s, h, h, (int64_t)s * h))) return rc;
    if ((rc = encode_map3(&tmPK, pkv, b, n_piv, h, 2 * (int64_t)h, (int64_t)n_piv * 2 * h))) return rc;
    if ((rc = encode_map3(&tmPV, pkv + h, b, n_piv, h, 2 * (int64_t)h, (int64_t)n_piv * 2 * h))) return rc;
    BwdParams p;
    p.b = b; p.heads = heads; p.s = s;
    p.sep_eff = 0;
    p.scale = 1.0f / sqrtf((float)head_dim);
    p.scale_log2 = p.scale * LOG2E;
    p.lse = lse; p.delta = delta; p.dq_acc = dq_acc;
    p.drop_scale = dropout_p > 0.f ? 1.0f / (1.0f - dropout_p) : 1.0f;
    const sparse::KeepLayout L = sparse::keep_layout(b, heads, s, n_piv, query_window, key_window_times);
    p.sp_w = query_window; p.sp_times = key_window_times;
    p.piv_bias_log2 = logf((float)(s / n_piv)) * LOG2E;
    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<MODE_BAND>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        CV_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<MODE_PIVOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set = true;
    }
    // band pass: dK / dV rows of the sequence
    p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
    p.sk = s; p.kv_rows = s; p.piv_pos = nullptr;
    p.drop_mask = dropout_p > 0.f ? drop_mask + L.fwd_words : nullptr;
    p.keep_rows = L.nkb * BLK; p.keep_slots = L.tq;
    attn_bwd_kernel<MODE_BAND><<<dim3((s + BLK - 1) / BLK, heads, b), NUM_THREADS, SMEM_BYTES, st>>>(tmQ, tmK, tmV, tmDO, p);
    CV_LAUNCH_CHECK();
    if (key_window_times * query_window < s) {       // some query sees pivots at all
        p.dqkv = dpiv;
        p.sk = n_piv; p.kv_rows = n_piv; p.piv_pos = pos32;
        p.drop_mask = dropout_p > 0.f ? drop_mask + L.fwd_words + L.band_words : nullptr;
        p.keep_rows = L.npb * BLK; p.keep_slots = L.np;
        attn_bwd_kernel<MODE_PIVOT><<<dim3((n_piv + BLK - 1) / BLK, heads, b), NUM_THREADS, SMEM_BYTES, st>>>(
            tmQ, tmPK, tmPV, tmDO, p);
        CV_LAUNCH_CHECK();
        scatter_pivot_grads_kernel<<<b * n_piv, 256, 0, st>>>(dpiv, pos32, static_cast<__nv_bfloat16*>(dqkv), n_piv, s, h);
        CV_LAUNCH_CHECK();
    }
    {
        const size_t rows = (size_t)b * s;
        const size_t n4 = rows * (h / 4);
        size_t blocks = (n4 + 255) / 256;
        size_t cap = (size_t)cvh::num_sms() * 8;
        attn_bwd_dq_store_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(
            dq_acc, static_cast<__nv_bfloat16*>(dqkv), rows, h);
        CV_LAUNCH_CHECK();
    }
    return 0;
}
