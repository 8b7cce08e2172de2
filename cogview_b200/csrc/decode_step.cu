// One autoregressive decode step (one new token per sequence, all layers + logits) as ONE persistent kernel.
//
// Reference path: generation/sampling.py:147-151 calling GPT2Model.forward (model/gpt2_modeling.py:106-123) with one
// token per sequence: per layer  LN1 -> QKV linear (mpu/layers.py:243) -> attention over the memory
// (mpu/sparse_transformer.py:652-673) -> dense (mpu/layers.py:319) -> x + LN3 -> LN2 -> h->4h + GELU -> 4h->h ->
// y + LN4 (mpu/sparse_transformer.py:314-342), then the final LayerNorm and the tied-embedding logits.
//
// The step is HBM bound: 7.86 GB of bf16 weights are read once per step (SURVEY §8(d)).  Launching one small kernel
// per linear leaves every launch in its ramp-up / drain, so:
//
//   * one CTA per SM, resident for the whole step: 16 consumer warps + 1 producer warp;
//   * every weight matrix is split into contiguous row ranges, one per CTA;
//   * the producer warp walks the CTA's static schedule (all matrices of all layers, the CTA's share of the K|V cache
//     after each QKV matrix, then the vocabulary matrix) and copies 16-row x KS-column slabs into a shared-memory ring
//     with cp.async.bulk (one bulk copy per weight row segment, >= 512 B contiguous, L2 evict-first) / TMA tiles for
//     K|V, completion on an mbarrier per stage.  Weights do not depend on activations, so the producer never waits for
//     a grid barrier: while the consumers sit in one of the 5 grid barriers of a layer the ring fills with the next
//     matrix;
//   * consumer warps split K inside a stage, feed mma.sync.m16n8k16 (weights = A, 16 output columns as rows;
//     activations = B, up to 8 sequences as columns) from shared memory with conflict-free 16-byte loads (row pitch
//     = 64 mod 128 bytes; the k-permutation of the fragments is the same for A and B, so a dot product is unchanged),
//     reduce the 16 partial tiles through shared memory and apply bias / GELU;
//   * the 4h->h product runs over four K chunks of h columns: the chunk's activations are copied (cp.async, next
//     chunk in flight behind the current one) into one of two operand buffers, the accumulators of the CTA's (<= 2)
//     row tiles stay in registers across the chunks — no split-K partials, no atomics, bf16 output like every other
//     linear;
//   * the fp32 residual stream never leaves the SM: every CTA keeps the full [M, h] stream in REGISTERS (20 floats per
//     thread at M <= 4) and computes the Sandwich-LN glue (two abs-max LayerNorms + residual,
//     mpu/sparse_transformer.py:40-44) redundantly straight into its shared-memory operand.  The only thing a glue reads
//     from other SMs is the bf16 output of the preceding linear (20 KB at M = 4), not the whole residual stream;
//   * attention over the K|V cache runs on (sequence, head, key-block) units, balanced over the CTAs as one flattened
//     range; a (sequence, head) pair that straddles CTAs is merged by the CTA that owns its FIRST key blocks — which
//     it processes LAST, so the other contributors' partial states (plain stores + one release-add) are already there:
//     no grid barrier, no atomic round trip on the critical path; the new token's K/V are appended in place;
//   * grid barrier = bar.sync; red.release.gpu; ld.acquire.gpu poll (one L2 round trip).
//
// Code size matters: the per-layer working set of the first versions did not fit the 32 KB L1.5 instruction cache (200
// KB of SASS, 3000 instructions of inlined 64-bit divisions) and every phase started with instruction fetches from an
// L2 that the weight stream keeps busy.  Row ranges are now computed once (32-bit), every heavy routine has one call
// site, slow paths are out of line.
//
// Everything exchanged between CTAs goes through L2 (ld.global.cg / cp.async.cg / st + release): L1 is not coherent
// and there is no kernel boundary to invalidate it.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;
typedef __nv_bfloat16 bf16;

constexpr int CW = 16;              // consumer warps: two groups of GW that take alternate ring stages
constexpr int GW = 8;               // warps per group = K slices of a stage
constexpr int CT = CW * 32;         // consumer threads
constexpr int NT = CT + 64;         // + one producer warp + one epilogue warp
constexpr int CE = CT + 32;         // consumers + epilogue warp (named barriers they share)
enum { BAR_CONS = 1, BAR_ATT = 2, BAR_PFULL = 3, BAR_PFREE = 5, BAR_ALL = 7 };   // named barrier ids (PFULL/PFREE: +pbuf)
constexpr int TILE = 16;            // weight rows (output columns) per MMA tile
constexpr int NQ_FC2 = 4;           // K chunks of the 4h->h matrix
constexpr int HD = 64;              // head dim
constexpr int NB = 16;              // mbarrier pairs of the ring = stages in flight (stages are variable-sized)
constexpr int MAXM = 8;
constexpr int KVB = 64;             // keys per K|V ring stage (16 warps x 4 keys)
constexpr int KVB_MAX = 64;         // key blocks per (sequence, head): max_len <= KVB * KVB_MAX = 4096
constexpr int PART_STRIDE = HD + 2; // attention partial: acc[64], m, l
constexpr int MAXSEG = 16;          // (sequence, head) segments of one CTA in the attention phase
enum { MAT_QKV = 0, MAT_DENSE = 1, MAT_FC1 = 2, MAT_FC2 = 3, MAT_WTE = 4 };
enum { EPI_BF16 = 0, EPI_BF16_GELU = 1, EPI_F32 = 2 };

struct Params {
    const cv_decode_layer* layers;
    int L, h, heads, V, M, max_len;
    float eps, eps_final;
    const bf16 *wte, *wpe, *lnf_g, *lnf_b;
    const int64_t *ids, *pos;
    const int* cur_len;
    bf16* cache;
    int64_t cache_ls, cache_bs;
    float* logits;
    int64_t ldl;
    // workspace
    bf16 *qkv, *ctx, *attn_out, *h4, *mlp_out;
    float* attn_part;
    unsigned int* attn_cnt;
    unsigned long long *bar_ctr, *bar_base;
    int* err;
    unsigned long long* prof;      // optional [grid][L][32]: globaltimer stamps of the phase boundaries + wait accounting
    // derived on the host
    int kstage, ring_bytes, pitch, xpitch, xbuf_bytes, dbg;
    float scale_log2;
};

// shared-memory carve-up (bytes from the 1024-aligned base)
constexpr int SM_BAR = 0;                                  // full[NB], empty[NB]
constexpr int SM_RNG = 2 * NB * 8;                         // int rng[5][2]: the CTA's row range of every matrix shape
constexpr int SM_ASZ = SM_RNG + 64;                        // uint32 asz[NB]: bytes held by the stage in each barrier slot
constexpr int SM_RED = 512;                                // float2 red[4][CW]
constexpr int SM_PART = SM_RED + 4 * CW * 8;               // float part[2][CW][TILE][8]  (attention: states + q|k|v)
constexpr int SM_XOP = ((SM_PART + 2 * CW * TILE * 8 * 4) + 127) / 128 * 128;
static_assert(CW * HD * 4 + MAXSEG * 3 * HD * 2 <= 2 * CW * TILE * 8 * 4, "attention staging must fit the tile partials");

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
__device__ __forceinline__ void tma_load_4d_u32(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                                int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
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
__device__ __forceinline__ float bflo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bfhi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ void bf16x8_to_float(const uint4& u, float (&f)[8]) {
    f[0] = bflo(u.x); f[1] = bfhi(u.x); f[2] = bflo(u.y); f[3] = bfhi(u.y);
    f[4] = bflo(u.z); f[5] = bfhi(u.z); f[6] = bflo(u.w); f[7] = bfhi(u.w);
}
__device__ __forceinline__ uint4 ldcg_u128(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }

// ---- waits: one try on the fast path, the bounded spin (wall-clock timeout -> trap the host sees) out of line ----
__device__ __noinline__ void wait_failed(int* err, int code) {
    if (err != nullptr) atomicExch(err, code);
    printf("cogview_b200: decode_step_kernel wait timed out (code %d, block %d, thread %d)\n", code, blockIdx.x,
           threadIdx.x);
    __trap();
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
__device__ __noinline__ void ring_wait_slow(uint32_t addr, uint32_t parity, int* err) {
    uint32_t spins = 0;
    uint64_t t0 = 0;
    while (!mbar_try(addr, parity)) {
        if ((++spins & 0x3ff) == 0) {
            const uint64_t now = global_timer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > CV_WAIT_TIMEOUT_NS) wait_failed(err, 1);
        }
    }
}
__device__ __forceinline__ void ring_wait(uint32_t addr, uint32_t parity, int* err) {
    if (!mbar_try(addr, parity)) ring_wait_slow(addr, parity, err);
}
// spin until *ctr >= target (acquire)
__device__ __noinline__ void poll_u64(const unsigned long long* ctr, unsigned long long target, int* err, int code) {
    uint32_t spins = 0;
    uint64_t t0 = 0;
    while (true) {
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ctr) : "memory");
        if (v >= target) return;
        if ((++spins & 0xff) == 0) {
            const uint64_t now = global_timer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > CV_WAIT_TIMEOUT_NS) wait_failed(err, code);
        }
    }
}
__device__ __noinline__ void poll_u32(const unsigned int* ctr, unsigned int target, int* err, int code) {
    uint32_t spins = 0;
    uint64_t t0 = 0;
    while (true) {
        unsigned int v;
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        if (v >= target) return;
        if ((++spins & 0xff) == 0) {
            const uint64_t now = global_timer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > CV_WAIT_TIMEOUT_NS) wait_failed(err, code);
        }
    }
}

template <int MR, int CPW>
__global__ void __launch_bounds__(NT, 1) decode_step_kernel(const __grid_constant__ Params p,
                                                            const __grid_constant__ CUtensorMap tmKV) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int cta = blockIdx.x, G = gridDim.x;
    const int h = p.h, M = p.M;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + SM_BAR);
    uint64_t* empty = full + NB;
    int* rng = reinterpret_cast<int*>(smem + SM_RNG);
    float* red = reinterpret_cast<float*>(smem + SM_RED);
    float* part = reinterpret_cast<float*>(smem + SM_PART);
    const uint32_t xop = smem_u32(smem + SM_XOP);
    const uint32_t ring = xop + 2 * p.xbuf_bytes;
    const uint32_t full0 = smem_u32(full), empty0 = smem_u32(empty);
    const int nks = h / p.kstage;

    if (tid == 0) {
        for (int i = 0; i < NB; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], CW);
        }
        fence_barrier_init();
        // row ranges [N cta / G, N (cta + 1) / G) of the five matrix shapes (N G < 2^32)
        const unsigned int c0 = (unsigned int)cta, gg = (unsigned int)G;
        const unsigned int Ns[5] = {3u * h, (unsigned int)h, 4u * h, (unsigned int)h, (unsigned int)p.V};
        for (int i = 0; i < 5; ++i) {
            rng[2 * i] = (int)((Ns[i] * c0) / gg);
            rng[2 * i + 1] = (int)((Ns[i] * (c0 + 1u)) / gg);
        }
    }
    __syncthreads();

    // ============================================================================================
    // producer warp: the weight / K|V stream
    // ============================================================================================
    if (warp == CW) {
        const uint64_t pol = evict_first_policy();
        const int t_p = __ldg(p.cur_len);
        const int nblk_p = (t_p + KVB - 1) / KVB;
        const unsigned int nbt_p = (unsigned int)(M * p.heads * nblk_p);
        const int kf0 = (int)((nbt_p * (unsigned int)cta) / (unsigned int)G);
        const int kf1 = (int)((nbt_p * (unsigned int)(cta + 1)) / (unsigned int)G);
        // The small parameters of a layer (LayerNorm vectors, biases: ~85 KB) are first-touch HBM reads on the
        // consumers' critical path; one CTA per layer pulls them into L2 a layer ahead.
        auto prefetch_params = [&](int l) {
            if (l >= p.L || cta != l % G || lane >= 16) return;
            const int f = lane;
            if (f == 2 || f == 4 || f == 10 || f == 12) return;          // the weight matrices
            const void* ptr = reinterpret_cast<const void* const*>(p.layers + l)[f];
            bulk_prefetch_l2(ptr, (uint32_t)h * 2u * (f == 3 ? 3u : (f == 11 ? 4u : 1u)));
        };
        prefetch_params(0);
        if (cta == G - 1 && lane < 2) bulk_prefetch_l2(lane == 0 ? p.lnf_g : p.lnf_b, (uint32_t)h * 2u);
        // The ring is a BYTE ring: a stage takes what it needs (16 rows x KS columns = 41 KB, the 1-2 leftover rows of
        // a row range 3-5 KB, a K|V tile pair 16 KB), so that the bytes in flight per SM do not depend on the stage mix
        // (with fixed 41 KB slots the 4h->h stream, whose stages alternate 16-row / 1-row tiles, and the K|V stream had
        // half / 40 % of the ring in flight and ran latency-bound).  Stage i signals on barrier pair i % NB; both sides
        // derive the same offsets from the same static schedule.
        volatile uint32_t* asz = reinterpret_cast<volatile uint32_t*>(smem + SM_ASZ);
        const uint32_t R = (uint32_t)p.ring_bytes;
        int si = 0, tail = 0;
        uint32_t off = 0, used = 0;
        auto alloc = [&](uint32_t size) -> uint32_t {
            const bool wrap = off + size > R;                            // a stage never wraps: skip the end of the ring
            const uint32_t pad = wrap ? R - off : 0u;
            const uint32_t need = size + pad;
            while (used + need > R || tail + NB <= si) {                 // wait for the oldest stages to be released
                ring_wait(empty0 + (tail & (NB - 1)) * 8, (uint32_t)(tail / NB) & 1u, p.err);
                used -= asz[tail & (NB - 1)];
                ++tail;
            }
            if (wrap) off = 0;
            asz[si & (NB - 1)] = need;
            const uint32_t a = ring + off;
            off += size;
            used += need;
            return a;
        };
        const int n_items = 4 * p.L + 1;
#pragma unroll 1
        for (int it = 0; it < n_items; ++it) {
            const int l = it >> 2, which = it & 3;
            const bool fin = it == n_items - 1;
            const bf16* W = p.wte;
            int64_t ldw = h;
            int mat = MAT_WTE, nq = 1;
            if (!fin) {
                if (which == 0) prefetch_params(l + 1);
                const int fld = which == 0 ? 2 : (which == 1 ? 4 : (which == 2 ? 10 : 12));
                W = reinterpret_cast<const bf16* const*>(p.layers + l)[fld];
                mat = which;
                if (which == 3) { ldw = 4 * (int64_t)h; nq = NQ_FC2; }
            }
            const int r0 = rng[2 * mat], r1 = rng[2 * mat + 1];
#pragma unroll 1
            for (int kq = 0; kq < nq; ++kq) {
#pragma unroll 1
                for (int r = r0; r < r1; r += TILE) {
                    const int rows = min(TILE, r1 - r);
                    const bf16* src = W + (size_t)(r + min(lane, rows - 1)) * ldw + (size_t)kq * h;
                    if (p.dbg & 1) src = W + (size_t)(r0 + min(lane, rows - 1)) * ldw;   // timing experiment: L2-hot source
#pragma unroll 1
                    const uint32_t wsize = (uint32_t)(rows * p.pitch + 127) & ~127u;
#pragma unroll 1
                    for (int ks = 0; ks < nks; ++ks) {
                        const uint32_t dst = alloc(wsize);
                        const int b = si & (NB - 1);
                        if (lane == 0) mbar_expect_tx(&full[b], (uint32_t)(rows * p.kstage * 2));
                        __syncwarp();
                        if (lane < rows)
                            bulk_g2s(dst + lane * p.pitch, src + ks * p.kstage, (uint32_t)(p.kstage * 2), full0 + b * 8, pol);
                        ++si;
                    }
                }
            }
            if (!fin && which == 0) {                      // this CTA's K|V key blocks of layer l follow its QKV weights
#pragma unroll 1
                for (int f = kf0; f < kf1; ++f) {
                    const int bh = f / nblk_p, blk = f - bh * nblk_p;
                    const int head = bh % p.heads, batch = bh / p.heads;
                    const uint32_t dst = alloc(2 * KVB * 128);
                    const int b = si & (NB - 1);
                    if (lane == 0) {
                        mbar_expect_tx(&full[b], 2 * KVB * 128);
                        tma_load_4d_u32(dst, &tmKV, full0 + b * 8, head * HD, blk * KVB, batch, l);
                        tma_load_4d_u32(dst + KVB * 128, &tmKV, full0 + b * 8, h + head * HD, blk * KVB, batch, l);
                    }
                    __syncwarp();
                    ++si;
                }
            }
        }
        return;
    }

    // the linear of phase `phs` of layer `l` (fin: the logits)
    struct Lin {
        int mat, nq, epi;
        const bf16 *bias, *xsrc;
        void* out;
        int64_t ldo, xld;
    };
    auto phase_linear = [&](bool fin, int l, int phs) -> Lin {
        Lin L;
        L.mat = MAT_WTE; L.nq = 1; L.epi = EPI_F32; L.bias = nullptr; L.xsrc = nullptr; L.out = p.logits; L.ldo = p.ldl; L.xld = h;
        if (!fin) {
            const cv_decode_layer& Lw = p.layers[l];
            L.epi = EPI_BF16;
            L.ldo = h;
            if (phs == 0) {
                L.mat = MAT_QKV; L.bias = static_cast<const bf16*>(Lw.b_qkv); L.out = p.qkv; L.ldo = 3 * h;
            } else if (phs == 2) {
                L.mat = MAT_DENSE; L.bias = static_cast<const bf16*>(Lw.b_dense); L.out = p.attn_out; L.xsrc = p.ctx;
            } else if (phs == 3) {
                L.mat = MAT_FC1; L.epi = EPI_BF16_GELU; L.bias = static_cast<const bf16*>(Lw.b_fc1); L.out = p.h4; L.ldo = 4 * h;
            } else {
                L.mat = MAT_FC2; L.nq = NQ_FC2; L.bias = static_cast<const bf16*>(Lw.b_fc2); L.out = p.mlp_out;
                L.xsrc = p.h4; L.xld = 4 * h;
            }
        }
        return L;
    };

    // ============================================================================================
    // epilogue warp: sums the 16 K-slice partials of every finished [16 outputs x 8 sequences] tile, applies bias /
    // GELU and stores — off the consumers' critical path (a CTA-wide bar.sync + reduce per tile would stall every
    // consumer warp).  part[pbuf] is handed over with named barriers:
    // consumers bar.arrive PFULL after writing, this warp bar.arrive PFREE after reading.
    // ============================================================================================
    if (warp == CW + 1) {
        named_bar_arrive(BAR_PFREE + 0, CE);
        named_bar_arrive(BAR_PFREE + 1, CE);
        const int nn = lane >> 1, mi0 = (lane & 1) * 4;
        int pbuf = 0, l = 0, phs = 0;
        const int n_it = 5 * p.L + 1;
#pragma unroll 1
        for (int it = 0; it < n_it; ++it) {
            const bool fin = it == n_it - 1;
            if (fin || phs != 1) {
                const Lin L = phase_linear(fin, l, phs);
                const int r0 = rng[2 * L.mat], r1 = rng[2 * L.mat + 1];
#pragma unroll 1
                for (int r = r0; r < r1; r += TILE) {
                    const int n = r + nn;
                    float bias_v = 0.f;
                    if (L.bias != nullptr) bias_v = __bfloat162float(L.bias[min(n, r1 - 1)]);
                    named_bar_sync(BAR_PFULL + pbuf, CE);
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int w = 0; w < CW; ++w) {
                        const float4 x = *reinterpret_cast<const float4*>(part + ((pbuf * CW + w) * TILE + nn) * 8 + mi0);
                        v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
                    }
                    named_bar_arrive(BAR_PFREE + pbuf, CE);
                    pbuf ^= 1;
                    if (n < r1) {
                        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int mi = mi0 + j;
                            if (mi < M) {
                                if (L.epi == EPI_F32) {
                                    static_cast<float*>(L.out)[(size_t)mi * L.ldo + n] = vv[j];
                                } else {
                                    float y = vv[j] + bias_v;
                                    if (L.epi == EPI_BF16_GELU) y = gelu_tanh(y);
                                    static_cast<bf16*>(L.out)[(size_t)mi * L.ldo + n] = __float2bfloat16_rn(y);
                                }
                            }
                        }
                    }
                }
            }
            if (!fin) {
                named_bar_sync(BAR_ALL, CE);               // this warp's stores are part of what the grid barrier releases
                if (++phs == 5) { phs = 0; ++l; }
            }
        }
        return;
    }

    // ============================================================================================
    // consumer warps
    // ============================================================================================
    const int g = lane >> 2, q = lane & 3;
    const int kpw = p.kstage / GW;                 // k elements per warp and stage ( = 32 * CPW )
    const int grp_w = warp / GW, wg = warp % GW;   // stage group, K slice inside a stage
    unsigned long long bar_target = *reinterpret_cast<volatile unsigned long long*>(p.bar_base);
    const int t_cached = __ldg(p.cur_len);         // tokens cached before this step; the new token sits at index t
    int pbuf = 0, sq = 0;                          // sq: stage counter (the producer's si)
    int prof_l = 0;
    uint32_t roff = 0;                             // read offset into the byte ring (same allocation rule as the producer)
    const uint32_t R = (uint32_t)p.ring_bytes;
    auto stage_addr = [&](uint32_t size) -> uint32_t {
        if (roff + size > R) roff = 0;
        const uint32_t a = ring + roff;
        roff += size;
        return a;
    };

    // rows >= M of the operand buffers stay zero for the whole kernel
    for (int i = tid; i < 2 * p.xbuf_bytes / 16; i += CT) sts128(xop + i * 16, make_uint4(0, 0, 0, 0));
    named_bar_sync(1, CT);

    auto stamp = [&](int l, int slot) {
        if (p.prof != nullptr && tid == 0) p.prof[((size_t)cta * p.L + l) * 32 + slot] = global_timer_ns();
    };
    auto grid_barrier = [&](int code) {
        named_bar_sync(BAR_ALL, CE);
        bar_target += (unsigned long long)G;
        if (tid == 0) {
            asm volatile("red.release.gpu.global.add.u64 [%0], %1;" ::"l"(p.bar_ctr), "l"(1ull) : "memory");
            poll_u64(p.bar_ctr, bar_target, p.err, code);
        }
        named_bar_sync(1, CT);
    };
    // asynchronous copy of M rows x h bf16 values (written by other CTAs) into an operand buffer
    auto xcopy = [&](const bf16* src, int64_t ld, uint32_t dst) {
        const int vpr = h >> 3;
#pragma unroll 1
        for (int mi = 0; mi < M; ++mi)
            for (int c = tid; c < vpr; c += CT) cp_async16(dst + mi * p.xpitch + c * 16, src + (size_t)mi * ld + c * 8);
    };

    // y[m, n] for the CTA's rows of one matrix.  Ring stages alternate between the two warp groups (stage counter `sq`
    // is the producer's), so two stages are in work at any time; every warp keeps its partial [16 x 8] tile and the 16
    // partials of a tile are summed through shared memory.  nq > 1 (the 4h->h matrix): K chunks of h columns, operand
    // chunk kq in buffer kq & 1 (chunk 0 requested by the caller), accumulators of the <= 2 row tiles carried in dA/dB.
    auto consume = [&](int mat, int nq, const bf16* xsrc, int64_t xld) {
        const int r0 = rng[2 * mat], r1 = rng[2 * mat + 1];
        const bool two_tiles = nq > 1 && r1 - r0 > TILE;
        long long c_wait = 0, c_bar = 0, c_tot = -clock64();   // wait accounting (tools/step_prof.py), prof runs only
        const bool acct = p.prof != nullptr && (tid == 0 || tid == 256);
        float dA[4] = {0.f, 0.f, 0.f, 0.f}, dB[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
        for (int kq = 0; kq < nq; ++kq) {
            uint32_t xb = xop;
            if (nq > 1) {
                cp_async_wait_all();                        // chunk kq has landed; every warp is done with chunk kq - 1
                named_bar_sync(1, CT);
                xb = xop + (kq & 1) * p.xbuf_bytes;
                if (kq + 1 < nq) xcopy(xsrc + (size_t)(kq + 1) * h, xld, xop + ((kq + 1) & 1) * p.xbuf_bytes);
            }
            const bool last = kq == nq - 1;
            // B fragments: the group's K stage index is the same for every tile of the chunk (2 stages per tile keep
            // the stage parity), so the activations are read from shared memory once per chunk, not once per stage
            const int ks_mine = nks == 1 ? 0 : (((sq & 1) == grp_w) ? 0 : 1);
            uint4 xv[CPW];
            {
                const uint32_t xa = xb + g * p.xpitch + (ks_mine * p.kstage + wg * kpw + q * 8) * 2;
#pragma unroll
                for (int c = 0; c < CPW; ++c) xv[c] = (MR == 8 || g < MR) ? lds128(xa + c * 64) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll 1
            for (int r = r0; r < r1; r += TILE) {
                const int rows = min(TILE, r1 - r);          // rows past the range are not in the stage: re-read the last one
                const uint32_t wsize = (uint32_t)(rows * p.pitch + 127) & ~127u;
                const uint32_t ra = min(g, rows - 1) * p.pitch + (wg * kpw + q * 8) * 2;
                const uint32_t rb = min(g + 8, rows - 1) * p.pitch + (wg * kpw + q * 8) * 2;
#pragma unroll 1
                for (int ks = 0; ks < nks; ++ks) {
                    const uint32_t sa = stage_addr(wsize);
                    const int b = sq & (NB - 1);
                    if ((sq & 1) == grp_w) {
                        if (acct) c_wait -= clock64();
                        ring_wait(full0 + b * 8, (uint32_t)(sq / NB) & 1u, p.err);
                        if (acct) c_wait += clock64();
                        if (!(p.dbg & 2)) {
                            uint4 w0[CPW], w1[CPW];
#pragma unroll
                            for (int c = 0; c < CPW; ++c) {
                                w0[c] = lds128(sa + ra + c * 64);
                                w1[c] = lds128(sa + rb + c * 64);
                            }
#pragma unroll
                            for (int c = 0; c < CPW; ++c) {
                                mma_16816(dA, w0[c].x, w1[c].x, w0[c].y, w1[c].y, xv[c].x, xv[c].y);
                                mma_16816(dA, w0[c].z, w1[c].z, w0[c].w, w1[c].w, xv[c].z, xv[c].w);
                            }
                        }
                        __syncwarp();
                    }
                    if (lane == 0) mbar_arrive(&empty[b]);   // (the other group's stage: nothing to read)
                    ++sq;
                }
                if (last) {
                    // D fragment: d0,d1 = (row g, cols 2q,2q+1), d2,d3 = (row g+8, ...); row = output column, col = sequence
                    if (acct) c_bar -= clock64();
                    named_bar_sync(BAR_PFREE + pbuf, CE);    // the epilogue warp has read this buffer (two tiles ago)
                    if (acct) c_bar += clock64();
                    float* pw = part + ((pbuf * CW + warp) * TILE) * 8;
                    pw[g * 8 + 2 * q] = dA[0];
                    pw[g * 8 + 2 * q + 1] = dA[1];
                    pw[(g + 8) * 8 + 2 * q] = dA[2];
                    pw[(g + 8) * 8 + 2 * q + 1] = dA[3];
                    dA[0] = dA[1] = dA[2] = dA[3] = 0.f;
                    named_bar_arrive(BAR_PFULL + pbuf, CE);
                    pbuf ^= 1;
                }
                if (two_tiles) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) { const float tmp = dA[i]; dA[i] = dB[i]; dB[i] = tmp; }
                }
            }
        }
        if (acct && mat < MAT_WTE) {
            unsigned long long* d = p.prof + ((size_t)cta * p.L + prof_l) * 32 + 16 + (tid == 0 ? 0 : 8) + mat * 2;
            d[0] = (unsigned long long)c_wait;
            d[1] = (unsigned long long)c_bar;
        }
        (void)c_tot;
    };

    // ------------------------------------------------------------------------------------------------
    // Sandwich-LN glue, computed redundantly by every CTA on the register-resident residual stream `res`:
    //   res += LN_post(gemm_out / (max|gemm_out| / 8))      (skipped when gemm_out == nullptr)
    //   xn   = LN_pre(res / (max|res| / 8))  -> operand buffer 0
    // Thread mapping: row = tid / TPR (TPR = 512 / MR threads per sequence), NVT 4-column vectors per thread.
    // ------------------------------------------------------------------------------------------------
    constexpr int TPR = CT / MR;
    constexpr int WPR = TPR / 32;
    constexpr int NVT = (2560 / 4 + TPR - 1) / TPR;
    const int hv = h >> 2;
    const float inv_h = 1.0f / h;
    const int grow = tid / TPR, gt = tid - grow * TPR;
    const bool row_ok = grow < M;
    float4 res[NVT];
    // vector j of this thread: column block gt + TPR j; the index is clamped so that every global load is unconditional
    auto okj = [&](int j) { return row_ok && gt + TPR * j < hv; };
    auto vcj = [&](int j) { return okj(j) ? gt + TPR * j : 0; };
    {   // the embedding of the new token: wte[ids] + wpe[pos]   (mpu/layers.py:117-133, mpu/sparse_transformer.py:522-523)
        const int rr = row_ok ? grow : 0;
        const uint2* wrow = reinterpret_cast<const uint2*>(p.wte + (size_t)__ldg(p.ids + rr) * h);
        const uint2* prow = reinterpret_cast<const uint2*>(p.wpe + (size_t)__ldg(p.pos + rr) * h);
#pragma unroll
        for (int j = 0; j < NVT; ++j) {
            const uint2 x = __ldg(wrow + vcj(j)), y = __ldg(prow + vcj(j));
            res[j] = okj(j) ? make_float4(bflo(x.x) + bflo(y.x), bfhi(x.x) + bfhi(y.x), bflo(x.y) + bflo(y.y),
                                         bfhi(x.y) + bfhi(y.y))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    float2* red2 = reinterpret_cast<float2*>(red);          // [4][CW] (sum, max)
    auto reduce = [&](float& s, float& mx, int which) {
        s = warp_sum(s);
        mx = warp_max(mx);
        if (lane == 0) red2[which * CW + warp] = make_float2(s, mx);
        named_bar_sync(1, CT);
        float t = 0.f, m2 = 0.f;
#pragma unroll
        for (int w = 0; w < WPR; ++w) t += red2[which * CW + grow * WPR + w].x;
#pragma unroll
        for (int w = 0; w < CW; ++w) m2 = fmaxf(m2, red2[which * CW + w].y);
        s = t;
        mx = m2;
    };
    auto sum4 = [](const float4& x) { return (x.x + x.y) + (x.z + x.w); };
    auto amax4 = [](const float4& x) { return fmaxf(fmaxf(fabsf(x.x), fabsf(x.y)), fmaxf(fabsf(x.z), fabsf(x.w))); };
    auto dev4 = [](const float4& x, float mean) {
        const float a0 = x.x - mean, a1 = x.y - mean, a2 = x.z - mean, a3 = x.w - mean;
        return (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    };
    auto glue = [&](const bf16* gemm_out, const bf16* g_post, const bf16* b_post, const bf16* g_pre, const bf16* b_pre,
                    float eps_post, float eps_pre, int prof_layer) {
        const int growc = row_ok ? grow : 0;
        if (gemm_out != nullptr) {
            float4 v[NVT];
            uint2 gp[NVT], bp[NVT];                         // requested with the data: bar.sync is a compiler barrier
            float s = 0.f, amax = 0.f;
#pragma unroll
            for (int j = 0; j < NVT; ++j) {
                gp[j] = __ldg(reinterpret_cast<const uint2*>(g_post) + vcj(j));
                bp[j] = __ldg(reinterpret_cast<const uint2*>(b_post) + vcj(j));
            }
#pragma unroll
            for (int j = 0; j < NVT; ++j) {
                const uint2 u = __ldcg(reinterpret_cast<const uint2*>(gemm_out) + growc * hv + vcj(j));
                v[j] = okj(j) ? make_float4(bflo(u.x), bfhi(u.x), bflo(u.y), bfhi(u.y)) : make_float4(0.f, 0.f, 0.f, 0.f);
                s += sum4(v[j]);
                amax = fmaxf(amax, amax4(v[j]));
            }
            reduce(s, amax, 0);
            if (prof_layer >= 0) stamp(prof_layer, 13);
            const float c = amax * 0.125f, mean = s * inv_h;
            float ss = 0.f, dummy = 0.f;
#pragma unroll
            for (int j = 0; j < NVT; ++j)
                if (okj(j)) ss += dev4(v[j], mean);
            reduce(ss, dummy, 1);
            const float rstd = rsqrtf(ss * inv_h + eps_post * c * c);
#pragma unroll
            for (int j = 0; j < NVT; ++j) {
                if (okj(j)) {
                    res[j].x += (v[j].x - mean) * rstd * bflo(gp[j].x) + bflo(bp[j].x);
                    res[j].y += (v[j].y - mean) * rstd * bfhi(gp[j].x) + bfhi(bp[j].x);
                    res[j].z += (v[j].z - mean) * rstd * bflo(gp[j].y) + bflo(bp[j].y);
                    res[j].w += (v[j].w - mean) * rstd * bfhi(gp[j].y) + bfhi(bp[j].y);
                }
            }
        }
        uint2 gq[NVT], bq[NVT];                             // LN_pre parameters: in flight during the two reductions below
#pragma unroll
        for (int j = 0; j < NVT; ++j) {
            gq[j] = __ldg(reinterpret_cast<const uint2*>(g_pre) + vcj(j));
            bq[j] = __ldg(reinterpret_cast<const uint2*>(b_pre) + vcj(j));
        }
        float s2 = 0.f, amax2 = 0.f;
#pragma unroll
        for (int j = 0; j < NVT; ++j) {
            s2 += sum4(res[j]);
            amax2 = fmaxf(amax2, amax4(res[j]));
        }
        reduce(s2, amax2, 2);
        if (prof_layer >= 0) stamp(prof_layer, 14);
        const float c2 = amax2 * 0.125f, mean2 = s2 * inv_h;
        float ss2 = 0.f, dummy2 = 0.f;
#pragma unroll
        for (int j = 0; j < NVT; ++j)
            if (okj(j)) ss2 += dev4(res[j], mean2);
        reduce(ss2, dummy2, 3);
        if (prof_layer >= 0) stamp(prof_layer, 15);
        const float rstd2 = rsqrtf(ss2 * inv_h + eps_pre * c2 * c2);
#pragma unroll
        for (int j = 0; j < NVT; ++j) {
            const uint2 gg = gq[j], bb = bq[j];
            const float4 x = res[j];
            const uint32_t lo = pack_bf16x2((x.x - mean2) * rstd2 * bflo(gg.x) + bflo(bb.x),
                                            (x.y - mean2) * rstd2 * bfhi(gg.x) + bfhi(bb.x));
            const uint32_t hi = pack_bf16x2((x.z - mean2) * rstd2 * bflo(gg.y) + bflo(bb.y),
                                            (x.w - mean2) * rstd2 * bfhi(gg.y) + bfhi(bb.y));
            if (okj(j))
                asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(xop + grow * p.xpitch + (gt + TPR * j) * 8), "r"(lo),
                             "r"(hi) : "memory");
        }
        named_bar_sync(1, CT);
    };

    // ------------------------------------------------------------------------------------------------
    // attention of the new token over keys 0..t (standard_attention for sq = 1).  The cached keys reach the CTA through
    // the same ring as the weights ([64 keys x 64 dims] K and V tiles of this CTA's share of the flattened (sequence,
    // head, key block) space, requested right after the QKV weights).  A stage is worked on by all 16 warps (4 keys per
    // warp, 8 lanes per key); a warp keeps its online-softmax state across the consecutive blocks of a (sequence, head)
    // pair, the 16 warp states are merged through shared memory at the end of the CTA's segment of the pair.
    // ------------------------------------------------------------------------------------------------
    auto attention = [&](int l) {
        bf16* cache_l = p.cache + (size_t)l * p.cache_ls;
        const int grp = lane >> 3, sub = lane & 7;
        const int t = t_cached;
        const int nblk = (t + KVB - 1) / KVB;
        const int pairs = M * p.heads;
        const unsigned int nbt = (unsigned int)(pairs * nblk), gg = (unsigned int)G;
        int f0 = 0, f1 = 0, bh0 = cta, nseg;
        if (nblk > 0) {
            f0 = (int)((nbt * (unsigned int)cta) / gg);
            f1 = (int)((nbt * (unsigned int)(cta + 1)) / gg);
            bh0 = f0 / nblk;
            nseg = f1 > f0 ? (f1 - 1) / nblk - bh0 + 1 : 0;
        } else {
            nseg = cta < pairs ? (pairs - cta + G - 1) / G : 0;       // empty cache: pairs round-robin
        }
        float* sm_acc = part;                                         // [CW][HD] warp states
        float* sm_ml = red;                                           // [CW][2]
        bf16* sm_qkv = reinterpret_cast<bf16*>(part + CW * HD);       // [MAXSEG][q | k_new | v_new][HD]
        if (tid < nseg * 24) {                                        // the new token's q, k, v of every local segment
            const int s = tid / 24, w = tid - s * 24, which = w >> 3, sb = w & 7;
            const int bh = nblk > 0 ? bh0 + s : cta + s * G;
            const int head = bh % p.heads, batch = bh / p.heads;
            *reinterpret_cast<uint4*>(sm_qkv + (s * 3 + which) * HD + sb * 8) =
                ldcg_u128(p.qkv + (size_t)batch * 3 * h + which * h + head * HD + sb * 8);
        }
        named_bar_sync(1, CT);
#pragma unroll 1
        for (int s = 0; s < nseg; ++s) {
            const int bh = nblk > 0 ? bh0 + s : cta + s * G;
            const int head = bh % p.heads, batch = bh / p.heads;
            int b_lo = 0, b_hi = 0, ncontrib = 1, my_idx = 0;
            bool tail = true;                                         // this CTA owns the pair's last key block
            if (nblk > 0) {
                b_lo = max(f0, bh * nblk);
                b_hi = min(f1, (bh + 1) * nblk);
                tail = b_hi == (bh + 1) * nblk;
                if (nbt >= gg) {                                      // contributors = consecutive CTAs first..last
                    // owner of flattened block f: the largest c with floor(nbt c / G) <= f
                    const unsigned int fa = (unsigned int)(bh * nblk), fb = fa + (unsigned int)nblk - 1u;
                    const int cf = min(G - 1, (int)(((fa + 1u) * gg - 1u) / nbt));
                    const int cl = min(G - 1, (int)(((fb + 1u) * gg - 1u) / nbt));
                    ncontrib = cl - cf + 1;
                    my_idx = cta - cf;
                } else {                                              // every non-empty CTA owns exactly one block
                    ncontrib = nblk;
                    my_idx = f0 - bh * nblk;
                }
            }
            float qf[8], m = -INFINITY, lsum = 0.f, acc[8];
            bf16x8_to_float(*reinterpret_cast<const uint4*>(sm_qkv + (s * 3) * HD + sub * 8), qf);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll 1
            for (int f = b_lo; f <= b_hi; ++f) {
                uint4 kr, vr;
                bool valid;
                if (f < b_hi) {
                    const int blk = f - bh * nblk;
                    const int b = sq & (NB - 1);
                    ring_wait(full0 + b * 8, (uint32_t)(sq / NB) & 1u, p.err);
                    const uint32_t ka = stage_addr(2 * KVB * 128) + (warp * 4 + grp) * 128 + sub * 16;
                    kr = lds128(ka);
                    vr = lds128(ka + KVB * 128);
                    valid = blk * KVB + warp * 4 + grp < t;
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[b]);
                    ++sq;
                } else {                                              // after the blocks: the new token (key index t)
                    if (!(tail && warp == 0)) break;
                    kr = *reinterpret_cast<const uint4*>(sm_qkv + (s * 3 + 1) * HD + sub * 8);
                    vr = *reinterpret_cast<const uint4*>(sm_qkv + (s * 3 + 2) * HD + sub * 8);
                    valid = grp == 0;
                    if (valid && t < p.max_len) {                     // append K | V in place
                        bf16* kdst = cache_l + (size_t)batch * p.cache_bs + (size_t)t * 2 * h + head * HD + sub * 8;
                        *reinterpret_cast<uint4*>(kdst) = kr;
                        *reinterpret_cast<uint4*>(kdst + h) = vr;
                    }
                }
                float kf[8];
                bf16x8_to_float(kr, kf);
                float sdot = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) sdot = fmaf(qf[i], kf[i], sdot);
                sdot += __shfl_xor_sync(0xffffffffu, sdot, 1);
                sdot += __shfl_xor_sync(0xffffffffu, sdot, 2);
                sdot += __shfl_xor_sync(0xffffffffu, sdot, 4);
                if (valid) {
                    const float sc = sdot * p.scale_log2;
                    const float mn = fmaxf(m, sc);
                    const float alpha = exp2f(m - mn), pr = exp2f(sc - mn);
                    float vf[8];
                    bf16x8_to_float(vr, vf);
                    m = mn;
                    lsum = lsum * alpha + pr;
#pragma unroll
                    for (int i = 0; i < 8; ++i) acc[i] = fmaf(pr, vf[i], acc[i] * alpha);
                }
            }
            // merge the warp's four key groups (lanes with the same `sub`)
#pragma unroll
            for (int off = 8; off <= 16; off <<= 1) {
                const float mo = __shfl_xor_sync(0xffffffffu, m, off);
                const float lo = __shfl_xor_sync(0xffffffffu, lsum, off);
                const float mn = fmaxf(m, mo);
                const float wa = (m == -INFINITY) ? 0.f : exp2f(m - mn);
                const float wb = (mo == -INFINITY) ? 0.f : exp2f(mo - mn);
                lsum = lsum * wa + lo * wb;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float ao = __shfl_xor_sync(0xffffffffu, acc[i], off);
                    acc[i] = acc[i] * wa + ao * wb;
                }
                m = mn;
            }
            if (grp == 0) {
#pragma unroll
                for (int i = 0; i < 8; ++i) sm_acc[warp * HD + sub * 8 + i] = acc[i];
                if (sub == 0) { sm_ml[2 * warp] = m; sm_ml[2 * warp + 1] = lsum; }
            }
            named_bar_sync(1, CT);
            if (tid < HD) {
                float Mx = -INFINITY;
#pragma unroll
                for (int w = 0; w < CW; ++w) Mx = fmaxf(Mx, sm_ml[2 * w]);
                float Ls = 0.f, A = 0.f;
#pragma unroll 4
                for (int w = 0; w < CW; ++w) {
                    const float mw = sm_ml[2 * w];
                    const float wgt = (mw == -INFINITY) ? 0.f : exp2f(mw - Mx);
                    Ls += sm_ml[2 * w + 1] * wgt;
                    A += sm_acc[w * HD + tid] * wgt;
                }
                bf16* o = p.ctx + (size_t)batch * h + head * HD;
                float* slot = p.attn_part + (size_t)bh * KVB_MAX * PART_STRIDE;
                if (ncontrib == 1) {
                    o[tid] = __float2bfloat16_rn(A / Ls);
                } else if (my_idx != 0) {
                    // not the merger: post the partial state.  This segment is the FIRST thing this CTA works on, the
                    // merger (owner of the pair's first blocks) gets to the pair LAST.
                    float* dst = slot + my_idx * PART_STRIDE;
                    dst[tid] = A;
                    if (tid == 0) { dst[HD] = Mx; dst[HD + 1] = Ls; }
                    __threadfence();
                    named_bar_sync(2, HD);
                    if (tid == 0)
                        asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p.attn_cnt + bh), "r"(1u) : "memory");
                } else {
                    if (tid == 0) poll_u32(p.attn_cnt + bh, (unsigned int)(ncontrib - 1), p.err, 2);
                    named_bar_sync(2, HD);
                    float M2 = Mx;                                    // merge in contributor order: deterministic
#pragma unroll 1
                    for (int c2 = 1; c2 < ncontrib; ++c2) M2 = fmaxf(M2, __ldcg(slot + c2 * PART_STRIDE + HD));
                    const float w0 = (Mx == -INFINITY) ? 0.f : exp2f(Mx - M2);
                    float L2 = Ls * w0, A2 = A * w0;
#pragma unroll 1
                    for (int c2 = 1; c2 < ncontrib; ++c2) {
                        const float ms = __ldcg(slot + c2 * PART_STRIDE + HD);
                        const float wgt = (ms == -INFINITY) ? 0.f : exp2f(ms - M2);
                        L2 += __ldcg(slot + c2 * PART_STRIDE + HD + 1) * wgt;
                        A2 += __ldcg(slot + c2 * PART_STRIDE + tid) * wgt;
                    }
                    o[tid] = __float2bfloat16_rn(A2 / L2);
                    if (tid == 0) p.attn_cnt[bh] = 0u;                // next use: the next layer, grid barriers away
                }
            }
            named_bar_sync(1, CT);                                    // sm_acc / sm_ml free for the next segment
        }
    };

    // ------------------------------------------------------------------------------------------------
    // the step: 5 phases per layer (each ends in a grid barrier), then final LayerNorm + logits
    //   0: x += LN4(mlp_out_prev) (layer 0: the embedding), LN1, QKV        1: attention over the K|V cache
    //   2: dense                3: x += LN3(attn_out), LN2, h->4h + GELU     4: 4h->h
    // ------------------------------------------------------------------------------------------------
    const int n_it = 5 * p.L + 1;
    int l = 0, phs = 0;
#pragma unroll 1
    for (int it = 0; it < n_it; ++it) {
        const bool fin = it == n_it - 1;
        prof_l = l < p.L ? l : p.L - 1;
        const cv_decode_layer& Lw = p.layers[fin ? p.L - 1 : l];
        if (!fin && phs == 0) stamp(l, 0);
        if (fin || phs == 0 || phs == 3) {
            const bf16 *gemm_out, *g_post, *b_post, *g_pre, *b_pre;
            float eps_pre = p.eps;
            if (fin) {
                gemm_out = p.mlp_out;
                g_post = static_cast<const bf16*>(Lw.ln4_g); b_post = static_cast<const bf16*>(Lw.ln4_b);
                g_pre = p.lnf_g; b_pre = p.lnf_b; eps_pre = p.eps_final;
            } else if (phs == 0) {
                const cv_decode_layer& Lp = p.layers[l > 0 ? l - 1 : 0];
                gemm_out = l > 0 ? p.mlp_out : nullptr;
                g_post = static_cast<const bf16*>(Lp.ln4_g); b_post = static_cast<const bf16*>(Lp.ln4_b);
                g_pre = static_cast<const bf16*>(Lw.ln1_g); b_pre = static_cast<const bf16*>(Lw.ln1_b);
            } else {
                gemm_out = p.attn_out;
                g_post = static_cast<const bf16*>(Lw.ln3_g); b_post = static_cast<const bf16*>(Lw.ln3_b);
                g_pre = static_cast<const bf16*>(Lw.ln2_g); b_pre = static_cast<const bf16*>(Lw.ln2_b);
            }
            glue(gemm_out, g_post, b_post, g_pre, b_pre, p.eps, eps_pre, (!fin && phs == 0 && l > 0) ? l : -1);
            if (!fin) stamp(l, phs == 0 ? 1 : 8);
        }
        if (!fin && phs == 1) {
            attention(l);
        } else {
            const Lin L = phase_linear(fin, l, phs);
            if (L.xsrc != nullptr) {                        // activation operand written by other CTAs
                xcopy(L.xsrc, L.xld, xop);
                if (L.nq == 1) {
                    cp_async_wait_all();
                    named_bar_sync(1, CT);
                }
            }
            consume(L.mat, L.nq, L.xsrc, L.xld);
        }
        if (!fin) {
            const int after_work = phs == 0 ? 2 : (phs == 1 ? 4 : (phs == 2 ? 6 : (phs == 3 ? 9 : 11)));
            stamp(l, after_work);
            grid_barrier(100 * (phs + 1) + l);
            stamp(l, after_work + 1);
            if (++phs == 5) { phs = 0; ++l; }
        }
    }
    if (cta == 0 && tid == 0) *p.bar_base = bar_target;
}

// workspace layout (bytes); the first WS_DATA bytes hold counters and must start zeroed
constexpr size_t WS_CTR = 0;        // bar_ctr u64, bar_base u64, err int
constexpr size_t WS_ATTNCNT = 320;  // u32[MAXM * heads]
constexpr size_t WS_DATA = 8192;
inline size_t al256(size_t x) { return (x + 255) / 256 * 256; }

struct WsLayout {
    size_t qkv, ctx, attn_out, h4, mlp_out, attn_part, total;
};
WsLayout ws_layout(int h, int heads) {
    WsLayout w;
    size_t o = WS_DATA;
    w.qkv = o; o += al256((size_t)MAXM * 3 * h * 2);
    w.ctx = o; o += al256((size_t)MAXM * h * 2);
    w.attn_out = o; o += al256((size_t)MAXM * h * 2);
    w.h4 = o; o += al256((size_t)MAXM * 4 * h * 2);
    w.mlp_out = o; o += al256((size_t)MAXM * h * 2);
    w.attn_part = o; o += al256((size_t)MAXM * heads * KVB_MAX * PART_STRIDE * 4);
    w.total = o;
    return w;
}

}  // namespace

extern "C" int64_t cv_decode_step_workspace_bytes(int hidden, int heads) {
    if (hidden <= 0 || heads <= 0) return -1;
    return (int64_t)ws_layout(hidden, heads).total;
}

extern "C" int cv_decode_step(const cv_decode_step_args* a, void* stream) {
    CV_REQUIRE(a != nullptr && a->layers && a->wte && a->wpe && a->lnf_g && a->lnf_b && a->ids && a->pos &&
                   a->cur_len && a->cache && a->logits && a->workspace,
               "null pointer");
    const int h = a->hidden, heads = a->heads, M = a->batch;
    CV_REQUIRE(M >= 1 && M <= MAXM, "cv_decode_step handles 1 <= batch <= 8 sequences");
    CV_REQUIRE(h > 0 && h % 256 == 0 && h <= 2560, "hidden must be a multiple of 256 and <= 2560");
    CV_REQUIRE(heads > 0 && heads * HD == h && heads <= (1024 / MAXM), "hidden must be heads * 64");
    CV_REQUIRE(a->num_layers >= 1 && a->vocab >= 1 && a->max_len >= 1 && a->ld_logits >= a->vocab, "bad sizes");
    CV_REQUIRE(a->max_len <= KVB * KVB_MAX, "max_len must be <= 4096");
    CV_REQUIRE(a->cache_batch_stride == (int64_t)a->max_len * 2 * h &&
                   a->cache_layer_stride == (int64_t)M * a->max_len * 2 * h &&
                   (reinterpret_cast<uintptr_t>(a->cache) & 15) == 0,
               "the K|V cache must be a contiguous [layers, batch, max_len, 2*hidden] bf16 tensor");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(a->workspace) & 255) == 0, "workspace must be 256-byte aligned");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = cvh::num_sms();
    // row ranges: every CTA owns >= 1 row of every matrix and <= 2 row tiles of the 4h->h matrix; the attention
    // staging holds <= MAXSEG (sequence, head) segments per CTA; 32-bit range arithmetic
    CV_REQUIRE(grid >= 8 && h >= grid && (h + grid - 1) / grid <= 2 * TILE, "unsupported SM count for this hidden size");
    CV_REQUIRE((M * heads + grid - 1) / grid + 2 <= MAXSEG, "too many (sequence, head) pairs per SM");
    CV_REQUIRE((int64_t)a->vocab * (grid + 1) < (1ll << 32), "vocabulary too large");

    Params p;
    p.layers = a->layers;
    p.L = a->num_layers; p.h = h; p.heads = heads; p.V = a->vocab; p.M = M; p.max_len = a->max_len;
    p.eps = a->eps; p.eps_final = a->eps_final;
    p.wte = static_cast<const bf16*>(a->wte); p.wpe = static_cast<const bf16*>(a->wpe);
    p.lnf_g = static_cast<const bf16*>(a->lnf_g); p.lnf_b = static_cast<const bf16*>(a->lnf_b);
    p.ids = a->ids; p.pos = a->pos; p.cur_len = a->cur_len;
    p.cache = static_cast<bf16*>(a->cache);
    p.cache_ls = a->cache_layer_stride; p.cache_bs = a->cache_batch_stride;
    p.logits = a->logits; p.ldl = a->ld_logits;
    p.prof = static_cast<unsigned long long*>(a->prof);
    char* ws = static_cast<char*>(a->workspace);
    const WsLayout w = ws_layout(h, heads);
    p.bar_ctr = reinterpret_cast<unsigned long long*>(ws + WS_CTR);
    p.bar_base = p.bar_ctr + 1;
    p.err = reinterpret_cast<int*>(ws + WS_CTR + 16);
    p.attn_cnt = reinterpret_cast<unsigned int*>(ws + WS_ATTNCNT);
    p.qkv = reinterpret_cast<bf16*>(ws + w.qkv); p.ctx = reinterpret_cast<bf16*>(ws + w.ctx);
    p.attn_out = reinterpret_cast<bf16*>(ws + w.attn_out); p.h4 = reinterpret_cast<bf16*>(ws + w.h4);
    p.mlp_out = reinterpret_cast<bf16*>(ws + w.mlp_out);
    p.attn_part = reinterpret_cast<float*>(ws + w.attn_part);

    // stage = 16 weight rows x kstage columns; kstage = the largest multiple of 256 dividing h that is <= 1280
    int kstage = 256;
    for (int k = 256; k <= 1280; k += 256)
        if (h % k == 0) kstage = k;
    p.kstage = kstage;
    p.pitch = kstage * 2 + 64;                       // 64 mod 128: conflict-free 16-byte fragment loads
    p.xpitch = h * 2 + 64;
    const int MR = M <= 4 ? 4 : 8;
    p.xbuf_bytes = (MR * p.xpitch + 127) / 128 * 128;
    const int fixed = SM_XOP + 2 * p.xbuf_bytes;
    int max_smem = 0, dev = 0;
    CV_CUDA(cudaGetDevice(&dev));
    CV_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    int ring_bytes = (max_smem - fixed - 1024) / 128 * 128;
    if (const char* e = getenv("COGVIEW_B200_STEP_RING_KB")) {       // experiments: a smaller ring
        const int cap = atoi(e) * 1024;
        if (cap >= 32 * 1024 && cap < ring_bytes) ring_bytes = cap;
    }
    {
        const char* d = getenv("COGVIEW_B200_STEP_DBG");   // timing experiments (tools/step_prof.py); results are wrong
        p.dbg = d ? atoi(d) : 0;
    }
    const int max_stage = TILE * p.pitch > 2 * KVB * 128 ? TILE * p.pitch : 2 * KVB * 128;
    CV_REQUIRE(ring_bytes >= 2 * ((max_stage + 127) / 128 * 128), "not enough shared memory for the weight ring");
    p.ring_bytes = ring_bytes;
    const size_t smem_bytes = (size_t)fixed + (size_t)ring_bytes;
    p.scale_log2 = (1.0f / sqrtf((float)HD)) * 1.4426950408889634f;

    // K|V cache as a 4-D tensor: [2h | max_len | batch | layer], boxes of [64 dims x KVB keys] (one head's K or V)
    alignas(64) CUtensorMap tmKV;
    {
        const uint64_t dims[4] = {(uint64_t)2 * h, (uint64_t)a->max_len, (uint64_t)M, (uint64_t)a->num_layers};
        const uint64_t str[3] = {(uint64_t)2 * h * 2, (uint64_t)a->cache_batch_stride * 2, (uint64_t)a->cache_layer_stride * 2};
        const uint32_t box[4] = {HD, KVB, 1, 1};
        int rc = cvh::encode_tmap(&tmKV, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, a->cache, dims, str, box, nullptr,
                                  cvh::Swizzle::None);
        if (rc) return rc;
    }
    typedef void (*KernelFn)(const Params, const CUtensorMap);
    KernelFn fn = nullptr;
    const int cpw = kstage / 256;
#define DS_PICK(MR_)                                                    \
    switch (cpw) {                                                      \
        case 1: fn = decode_step_kernel<MR_, 1>; break;                 \
        case 2: fn = decode_step_kernel<MR_, 2>; break;                 \
        case 3: fn = decode_step_kernel<MR_, 3>; break;                 \
        case 4: fn = decode_step_kernel<MR_, 4>; break;                 \
        default: fn = decode_step_kernel<MR_, 5>; break;                \
    }
    if (MR == 4) { DS_PICK(4) } else { DS_PICK(8) }
#undef DS_PICK
    CV_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    static int coop = -1;
    if (coop < 0) {
        const char* e = getenv("COGVIEW_B200_COOP");
        int sup = 0;
        cudaDeviceGetAttribute(&sup, cudaDevAttrCooperativeLaunch, dev);
        coop = (sup && !(e && e[0] == '0')) ? 1 : 0;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(NT);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = coop ? 1 : 0;
    CV_CUDA(cudaLaunchKernelEx(&cfg, fn, p, tmKV));
    cvh::count_launches(1);
    return 0;
}
