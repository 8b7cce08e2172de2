// The operand ring of the persistent wgmma GEMM (csrc/gemm.cu), shared with the kernels that keep its main loop and
// replace its epilogue (csrc/vocab_logprob.cu).
//
//   warpgroup 0     TMA producer (one thread): load_tile streams a tile's k-blocks of A and B into a ring of
//                   128B-swizzled stages, each guarded by a full / empty mbarrier pair
//   warpgroups 1-2  wgmma consumers: mma_tile runs one 128 x width tile (each warpgroup owns 64 of its rows) into fp32
//                   register accumulators and hands every stage back as soon as its MMAs have retired
// Producer and consumers walk the same tile sequence, each with its own RingPos.
#pragma once
#include "common.cuh"

namespace cv {
namespace ring {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int NUM_THREADS = 384;

template <int BN>
struct Cfg {
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (BN == 256) ? 4 : 6;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

struct RingPos {
    int stage = 0;
    uint32_t phase = 0;
    template <int STAGES>
    __device__ __forceinline__ void advance() {
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
};

// The ring in dynamic shared memory: stages 1024-byte aligned, then full_bar[STAGES] and empty_bar[STAGES].
template <int BN>
struct Ring {
    uint8_t* smem;
    uint64_t* full_bar;     // one arrive (the producer's expect_tx) + the TMA bytes
    uint64_t* empty_bar;    // one arrive per consumer warp
    __device__ __forceinline__ explicit Ring(uint8_t* smem_raw) {
        smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
        full_bar = reinterpret_cast<uint64_t*>(smem + Cfg<BN>::STAGES * Cfg<BN>::STAGE_BYTES);
        empty_bar = full_bar + Cfg<BN>::STAGES;
    }
    // thread 0, followed by a __syncthreads() of the caller
    __device__ __forceinline__ void init(const CUtensorMap* tmA, const CUtensorMap* tmB) const {
        tma_prefetch_desc(tmA);
        tma_prefetch_desc(tmB);
        for (int i = 0; i < Cfg<BN>::STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);
        }
        fence_barrier_init();
    }
};

// Producer thread: the k-blocks of tile (m0, n0) of the given width (BN or BN / 2).  K-major operands are boxes of
// [rows x 64] (B in 128-row boxes), MN-major ones [64 x 64] boxes.
template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void load_tile(const Ring<BN>& r, RingPos& pos, const CUtensorMap* tmA,
                                          const CUtensorMap* tmB, int m0, int n0, int width, int num_k_blocks) {
    using C = Cfg<BN>;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait<false>(&r.empty_bar[pos.stage], pos.phase ^ 1);
        uint8_t* sA = r.smem + pos.stage * C::STAGE_BYTES;
        uint8_t* sB = sA + C::A_BYTES;
        mbar_expect_tx(&r.full_bar[pos.stage], C::A_BYTES + width * BK * 2);
        if (!A_MN) {
            tma_load_2d(sA, tmA, &r.full_bar[pos.stage], kb * BK, m0);
        } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
                tma_load_2d(sA + i * (BK * 128), tmA, &r.full_bar[pos.stage], m0 + i * 64, kb * BK);
        }
        if (!B_MN) {    // boxes of 128 rows: one per half tile
#pragma unroll
            for (int i = 0; i < BN / 128; ++i)
                if (i * 128 < width)
                    tma_load_2d(sB + i * (128 * BK * 2), tmB, &r.full_bar[pos.stage], kb * BK, n0 + i * 128);
        } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
                if (i * 64 < width)
                    tma_load_2d(sB + i * (BK * 128), tmB, &r.full_bar[pos.stage], n0 + i * 64, kb * BK);
        }
        pos.advance<C::STAGES>();
    }
}

template <int N, int TA, int TB>
__device__ __forceinline__ void mma_n(float* acc, uint64_t da, uint64_t db, uint32_t sc) {
    if constexpr (N == 256) wgmma_ss_n256<TA, TB>(*reinterpret_cast<float(*)[128]>(acc), da, db, sc);
    else if constexpr (N == 128) wgmma_ss_n128<TA, TB>(*reinterpret_cast<float(*)[64]>(acc), da, db, sc);
    else wgmma_ss_n64<TA, TB>(*reinterpret_cast<float(*)[32]>(acc), da, db, sc);
}

// Consumer warpgroup `half` (0 or 1): acc = rows 64 half .. 64 half + 63 of the tile times its columns (all BN, or
// the first BN / 2 when !full).  On return every MMA has retired and every stage of the tile is handed back.
// Fragment layout of acc: see common.cuh (d[4i + 2h + e]: row 16 warp + lane / 4 + 8h, column 8i + 2 (lane % 4) + e).
template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void mma_tile(const Ring<BN>& r, RingPos& pos, float (&acc)[BN / 2], int half, int lane,
                                         bool full, int num_k_blocks) {
    using C = Cfg<BN>;
    // K-major: 8-row groups 1024 B apart. MN-major: 64-element chunks one TMA box (BK*128 B) apart,
    // 8-row K groups 1024 B apart.
    constexpr uint32_t A_LBO = A_MN ? BK * 128 : 0, B_LBO = B_MN ? BK * 128 : 0;
    constexpr uint32_t A_KSTEP = A_MN ? 16 * 128 : 32, B_KSTEP = B_MN ? 16 * 128 : 32;
    const uint32_t a_half = A_MN ? half * (BK * 128) : half * (64 * 128);
    constexpr int TA = A_MN ? 1 : 0, TB = B_MN ? 1 : 0;
    int prev = -1;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait<false>(&r.full_bar[pos.stage], pos.phase);
        const uint32_t a_addr = smem_u32(r.smem + pos.stage * C::STAGE_BYTES) + a_half;
        const uint32_t b_addr = smem_u32(r.smem + pos.stage * C::STAGE_BYTES + C::A_BYTES);
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
            const uint64_t da = make_smem_desc_sw128(a_addr + k * A_KSTEP, A_LBO, 1024);
            const uint64_t db = make_smem_desc_sw128(b_addr + k * B_KSTEP, B_LBO, 1024);
            const uint32_t sc = (kb | k) != 0 ? 1u : 0u;
            if (full) mma_n<BN, TA, TB>(acc, da, db, sc);
            else mma_n<BN / 2, TA, TB>(acc, da, db, sc);
        }
        wgmma_commit();
        wgmma_wait<1>();                            // the previous k-block's MMAs retired: free its slot
        if (prev >= 0 && lane == 0) mbar_arrive(&r.empty_bar[prev]);
        prev = pos.stage;
        pos.advance<C::STAGES>();
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (lane == 0) mbar_arrive(&r.empty_bar[prev]);
}

}  // namespace ring
}  // namespace cv
