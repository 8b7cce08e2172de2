// cv_gemm_bf16: C[M,N] = op(A)[M,K] * op(B)[N,K]^T (+ bias) (+ tanh-GELU), bf16 operands, fp32 accumulate.
//
// Replaces the cuBLAS GEMMs the reference reaches through F.linear:
//   ColumnParallelLinear.forward  /root/reference/mpu/layers.py:239-249   (QKV, h->4h: bias fused)
//   RowParallelLinear.forward     /root/reference/mpu/layers.py:312-326   (out-proj, 4h->h: bias fused)
//   gelu_impl                     /root/reference/mpu/sparse_transformer.py:172-176 (fused epilogue)
//   logits GEMM                   /root/reference/model/gpt2_modeling.py:117-118
// and their autograd backward (dgrad: B MN-major; wgrad: A and B MN-major).
//
// Design (sm_90a): persistent, one CTA per SM, 3 warpgroups.
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor tiles -> 128B-swizzled smem ring (4-6 stages)
//   warpgroups 1-2  wgmma consumers: each owns 64 rows of the 128-row tile (m64 x BN x k16, fp32 accumulators in
//                   registers), then applies bias / activation / dropout / abs-max and stores its rows straight to
//                   global memory while the producer already streams the next tile's operands into the ring
#include <cstdlib>

#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {

using namespace cv;

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

struct GemmParams {
    int M, N, K;
    int num_m_blocks, num_n_blocks, num_k_blocks;
    int split_from;             // tiles [0, split_from) are BN wide; each later BN-wide tile is walked as two BN/2 halves
    int num_tiles;              // split_from + 2 * (number of split tiles)
    const __nv_bfloat16* bias;  // [N] or null
    int act;                    // 0 none, 1 tanh-GELU, 2 ReLU, 3 multiply by gelu'(aux) (GELU backward fused in dgrad)
    const __nv_bfloat16* aux;   // act == 3: pre-activation values [M, N] (leading dimension ldc)
    float* absmax;              // null or scalar: atomicMax |C| over valid entries
    int has_c2;                 // second bf16 output = pre-activation (bias added, no activation)
    DropoutArgs drop;           // drop.p > 0: output dropout after bias/activation (element index m*N + n)
    void* c;                    // output [M, N] (bf16 or fp32), leading dimension ldc
    __nv_bfloat16* c2;          // optional pre-activation output (bf16, same ldc)
    int64_t ldc;
};

// Tail-wave splitting: with T tiles on G persistent CTAs the last T % G tiles would occupy a whole wave while most
// SMs idle (34 x 10 = 340 tiles of a 4352 x 2560 output on 132 SMs: 2.6 waves cost 3).  When those r tiles fit twice
// (2r <= G) they are issued as 2r half-width tiles instead, so the last wave costs one half tile.
struct TileCoord { int m0, n0, width; };
template <int BN>
__device__ __forceinline__ TileCoord tile_coord(const GemmParams& p, int tile) {
    TileCoord t;
    if (tile < p.split_from) {
        t.m0 = (tile % p.num_m_blocks) * BM;
        t.n0 = (tile / p.num_m_blocks) * BN;
        t.width = BN;
    } else {
        const int h = tile - p.split_from;
        const int big = p.split_from + (h >> 1);
        t.m0 = (big % p.num_m_blocks) * BM;
        t.n0 = (big / p.num_m_blocks) * BN + (h & 1) * (BN / 2);
        t.width = BN / 2;
    }
    return t;
}

// dropout4 for the two consecutive elements idx, idx + 1 (idx even) that one accumulator fragment holds: the same
// Philox call (counter idx / 4), words x, y or z, w
__device__ __forceinline__ void dropout2(const DropoutArgs& d, uint64_t idx, float& a, float& b) {
    const uint4 r = philox4x32_10(d.seed, idx >> 2, d.stream);
    const uint32_t ra = (idx & 2) ? r.z : r.x, rb = (idx & 2) ? r.w : r.y;
    a = ra >= d.threshold ? a * d.scale : 0.f;
    b = rb >= d.threshold ? b * d.scale : 0.f;
}

template <int N, int TA, int TB>
__device__ __forceinline__ void mma_n(float* acc, uint64_t da, uint64_t db, uint32_t sc) {
    if constexpr (N == 256) wgmma_ss_n256<TA, TB>(*reinterpret_cast<float(*)[128]>(acc), da, db, sc);
    else if constexpr (N == 128) wgmma_ss_n128<TA, TB>(*reinterpret_cast<float(*)[64]>(acc), da, db, sc);
    else wgmma_ss_n64<TA, TB>(*reinterpret_cast<float(*)[32]>(acc), da, db, sc);
}

__device__ __forceinline__ void store_pair(__nv_bfloat16* dst, float a, float b, bool pair) {
    if (pair) *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(a, b);
    else dst[0] = __float2bfloat16_rn(a);
}
__device__ __forceinline__ void store_pair(float* dst, float a, float b, bool pair) {
    if (pair) *reinterpret_cast<float2*>(dst) = make_float2(a, b);
    else dst[0] = a;
}

template <int BN, bool A_MN, bool B_MN, bool OUT_F32>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    using C = Cfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
    uint64_t* full_bar = bars;                       // [STAGES]
    uint64_t* empty_bar = bars + C::STAGES;          // [STAGES]: one arrive per consumer warp

    const int wg = threadIdx.x >> 7;
    const int tid = threadIdx.x & 127;
    const int num_tiles = p.num_tiles;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < C::STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------ TMA producer ------------------------------
        setmaxnreg_dec<40>();
        if (tid == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const TileCoord tc = tile_coord<BN>(p, tile);
                const int m0 = tc.m0, n0 = tc.n0;
                for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                    mbar_wait<false>(&empty_bar[stage], phase ^ 1);
                    uint8_t* sA = smem + stage * C::STAGE_BYTES;
                    uint8_t* sB = sA + C::A_BYTES;
                    mbar_expect_tx(&full_bar[stage], C::A_BYTES + tc.width * BK * 2);
                    if (!A_MN) {
                        tma_load_2d(sA, &tmA, &full_bar[stage], kb * BK, m0);
                    } else {
#pragma unroll
                        for (int i = 0; i < BM / 64; ++i)
                            tma_load_2d(sA + i * (BK * 128), &tmA, &full_bar[stage], m0 + i * 64, kb * BK);
                    }
                    if (!B_MN) {    // boxes of 128 rows: one per half tile
#pragma unroll
                        for (int i = 0; i < BN / 128; ++i)
                            if (i * 128 < tc.width)
                                tma_load_2d(sB + i * (128 * BK * 2), &tmB, &full_bar[stage], kb * BK, n0 + i * 128);
                    } else {
#pragma unroll
                        for (int i = 0; i < BN / 64; ++i)
                            if (i * 64 < tc.width)
                                tma_load_2d(sB + i * (BK * 128), &tmB, &full_bar[stage], n0 + i * 64, kb * BK);
                    }
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ------------------------------ wgmma consumers + epilogue ------------------------------
        setmaxnreg_inc<232>();
        const int half = wg - 1;                            // rows 64 half .. 64 half + 63 of the tile
        const int warp = tid >> 5, lane = tid & 31;
        const int r_in = 64 * half + 16 * warp + (lane >> 2);   // this thread's rows: r_in and r_in + 8
        const int c_in = 2 * (lane & 3);                    // and columns 8i + c_in, + 1
        // K-major: 8-row groups 1024 B apart. MN-major: 64-element chunks one TMA box (BK*128 B) apart,
        // 8-row K groups 1024 B apart.
        constexpr uint32_t A_LBO = A_MN ? BK * 128 : 0, B_LBO = B_MN ? BK * 128 : 0;
        constexpr uint32_t A_KSTEP = A_MN ? 16 * 128 : 32, B_KSTEP = B_MN ? 16 * 128 : 32;
        const uint32_t a_half = A_MN ? half * (BK * 128) : half * (64 * 128);
        constexpr int TA = A_MN ? 1 : 0, TB = B_MN ? 1 : 0;
        int stage = 0;
        uint32_t phase = 0;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const TileCoord tc = tile_coord<BN>(p, tile);
            const bool full = tc.width == BN;
            int prev = -1;
            for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                mbar_wait<false>(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem + stage * C::STAGE_BYTES) + a_half;
                const uint32_t b_addr = smem_u32(smem + stage * C::STAGE_BYTES + C::A_BYTES);
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
                if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
                prev = stage;
                if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (lane == 0) mbar_arrive(&empty_bar[prev]);

            const int m0 = tc.m0, n0 = tc.n0;
            float tmax = 0.f;
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
                if (i * 8 >= tc.width) break;
                const int col = n0 + 8 * i + c_in;
                if (col >= p.N) continue;
                const bool pair = col + 1 < p.N;
                float b0 = 0.f, b1 = 0.f;
                if (p.bias != nullptr) {
                    b0 = __bfloat162float(p.bias[col]);
                    if (pair) b1 = __bfloat162float(p.bias[col + 1]);
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = m0 + r_in + 8 * h;
                    if (row >= p.M) continue;
                    float v0 = acc[4 * i + 2 * h] + b0, v1 = acc[4 * i + 2 * h + 1] + b1;
                    const size_t off = (size_t)row * p.ldc + col;
                    if (p.has_c2) store_pair(p.c2 + off, v0, v1, pair);     // pre-activation copy (bf16)
                    if (p.act == 1) {
                        v0 = gelu_tanh_fast(v0); v1 = gelu_tanh_fast(v1);
                    } else if (p.act == 2) {
                        v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
                    } else if (p.act == 3) {
                        v0 *= gelu_tanh_grad(__bfloat162float(p.aux[off]));
                        if (pair) v1 *= gelu_tanh_grad(__bfloat162float(p.aux[off + 1]));
                    }
                    if (p.drop.p > 0.f) dropout2(p.drop, (uint64_t)row * p.N + col, v0, v1);
                    if (OUT_F32) {
                        store_pair(static_cast<float*>(p.c) + off, v0, v1, pair);
                    } else {
                        store_pair(static_cast<__nv_bfloat16*>(p.c) + off, v0, v1, pair);
                        v0 = bf16_round(v0); v1 = bf16_round(v1);
                    }
                    if (p.absmax != nullptr) tmax = fmaxf(tmax, fmaxf(fabsf(v0), pair ? fabsf(v1) : 0.f));
                }
            }
            if (p.absmax != nullptr) {
                tmax = warp_max(tmax);
                if (lane == 0 && tmax > 0.f) atomic_max_nonneg(p.absmax, tmax);
            }
        }
    }
}

template <int BN, bool A_MN, bool B_MN, bool OUT_F32>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t stream) {
    auto kern = gemm_kernel<BN, A_MN, B_MN, OUT_F32>;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM_BYTES);
        if (e != cudaSuccess) return cvh::fail_cuda("cv_gemm_bf16", e);
        attr_set = true;
    }
    int tiles = p.num_tiles;
    int grid = tiles < cvh::gemm_sms() ? tiles : cvh::gemm_sms();
    kern<<<grid, NUM_THREADS, Cfg<BN>::SMEM_BYTES, stream>>>(tmA, tmB, p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cvh::fail_cuda("cv_gemm_bf16", e);
    cvh::count_launches(1);
    return 0;
}

template <int BN>
int dispatch(int a_mn, int b_mn, int out_f32, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p,
             cudaStream_t s) {
    if (out_f32) {
        if (!a_mn && !b_mn) return launch<BN, false, false, true>(tmA, tmB, p, s);
        if (!a_mn && b_mn) return launch<BN, false, true, true>(tmA, tmB, p, s);
        if (a_mn && b_mn) return launch<BN, true, true, true>(tmA, tmB, p, s);
        return cvh::fail_arg("cv_gemm_bf16", "A MN-major with B K-major is not instantiated");
    }
    if (!a_mn && !b_mn) return launch<BN, false, false, false>(tmA, tmB, p, s);
    if (!a_mn && b_mn) return launch<BN, false, true, false>(tmA, tmB, p, s);
    if (a_mn && b_mn) return launch<BN, true, true, false>(tmA, tmB, p, s);
    return cvh::fail_arg("cv_gemm_bf16", "A MN-major with B K-major is not instantiated");
}

}  // namespace

static bool split_tail_enabled() {   // COGVIEW_B200_GEMM_SPLIT_TAIL=0 disables tail-wave splitting (A/B measurements)
    static const bool on = [] {
        const char* e = getenv("COGVIEW_B200_GEMM_SPLIT_TAIL");
        return !(e && e[0] == '0');
    }();
    return on;
}

static int gemm_impl(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major, int64_t ldb,
                     void* Cout, int c_is_f32, int64_t ldc, void* C2, const void* bias, int act, float* absmax,
                     int M, int N, int K, int block_n, const cvh::HostDropout& hd, void* stream) {
    CV_REQUIRE(A && B && Cout, "null operand");
    CV_REQUIRE(M > 0 && N > 0 && K > 0, "M, N, K must be positive");
    CV_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "lda/ldb must be multiples of 8 elements (16-byte TMA strides)");
    CV_REQUIRE(c_is_f32 ? (ldc % 4 == 0) : (ldc % 8 == 0), "ldc must give 16-byte aligned rows");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(Cout) & 15) == 0,
               "operands must be 16-byte aligned");
    CV_REQUIRE(act >= 0 && act <= 3, "act must be 0 (none), 1 (tanh-GELU), 2 (ReLU) or 3 (x gelu'(aux))");
    CV_REQUIRE(act != 3 || (C2 != nullptr && !c_is_f32), "act 3 takes the pre-activation tensor through C2 (bf16 C)");
    CV_REQUIRE(!(C2 && c_is_f32), "pre-activation output requires bf16 C");
    cudaStream_t s = static_cast<cudaStream_t>(stream);

    int BN = block_n;
    if (BN == 0) {
        // Estimated time = waves x per-tile cost.  A 128x128 tile streams as many operand bytes per output column as
        // a 128x256 tile streams for two, so it is modelled at 3/4 of the wide tile's cost: 192 vs 256 per tile.
        // With tail-wave splitting (tile_coord) the last partial wave of the 256-wide schedule costs one 128-wide
        // tile when its tiles fit twice on the SMs.
        const int sms = cvh::gemm_sms();
        const int mb = (M + BM - 1) / BM;
        const long t128 = (long)mb * ((N + 127) / 128), t256 = (long)mb * ((N + 255) / 256);
        const long cost128 = (t128 + sms - 1) / sms * 192;
        const long r256 = t256 % sms;
        const long cost256 = t256 / sms * 256 + (r256 == 0 ? 0 : (2 * r256 <= sms ? 192 : 256));
        BN = cost128 < cost256 ? 128 : 256;
    }
    CV_REQUIRE(BN == 128 || BN == 256, "block_n must be 0 (auto), 128 or 256");

    GemmParams p;
    p.M = M; p.N = N; p.K = K;
    p.num_m_blocks = (M + BM - 1) / BM;
    p.num_n_blocks = (N + BN - 1) / BN;
    p.num_k_blocks = (K + BK - 1) / BK;
    {
        const int tiles = p.num_m_blocks * p.num_n_blocks, sms = cvh::gemm_sms();
        const int r = tiles % sms;
        const int nsplit = (BN == 256 && split_tail_enabled() && r > 0 && 2 * r <= sms) ? r : 0;
        p.split_from = tiles - nsplit;
        p.num_tiles = tiles + nsplit;
    }
    p.bias = static_cast<const __nv_bfloat16*>(bias);
    p.act = act;
    p.absmax = absmax;
    CV_REQUIRE(hd.p >= 0.f && hd.p < 1.f, "dropout probability must be in [0, 1)");
    CV_REQUIRE(hd.p == 0.f || N % 4 == 0, "dropout needs N % 4 == 0");
    p.drop.p = hd.p; p.drop.scale = hd.scale; p.drop.threshold = hd.threshold; p.drop.stream = hd.stream;
    p.drop.seed = hd.seed;
    p.has_c2 = C2 != nullptr && act != 3;
    p.aux = act == 3 ? static_cast<const __nv_bfloat16*>(C2) : nullptr;
    p.c = Cout;
    p.c2 = static_cast<__nv_bfloat16*>(C2);
    p.ldc = ldc;

    alignas(64) CUtensorMap tmA, tmB;
    int rc;
    // K-major: stored [rows = M or N, cols = K], box [tile rows x 64]. MN-major: stored [K, M or N], box [64 x 64].
    rc = a_mn_major ? cvh::encode_tmap_2d_bf16(&tmA, A, K, M, lda, BK, 64)
                    : cvh::encode_tmap_2d_bf16(&tmA, A, M, K, lda, BM, BK);
    if (rc) return rc;
    rc = b_mn_major ? cvh::encode_tmap_2d_bf16(&tmB, B, K, N, ldb, BK, 64)
                    : cvh::encode_tmap_2d_bf16(&tmB, B, N, K, ldb, 128, BK);   // 128-row boxes: BN / 128 per stage
    if (rc) return rc;
    if (BN == 256) return dispatch<256>(a_mn_major, b_mn_major, c_is_f32, tmA, tmB, p, s);
    return dispatch<128>(a_mn_major, b_mn_major, c_is_f32, tmA, tmB, p, s);
}

extern "C" int cv_gemm_bf16(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major, int64_t ldb,
                            void* Cout, int c_is_f32, int64_t ldc, void* C2, const void* bias, int act, float* absmax,
                            int M, int N, int K, int block_n, void* stream) {
    return gemm_impl(A, a_mn_major, lda, B, b_mn_major, ldb, Cout, c_is_f32, ldc, C2, bias, act, absmax, M, N, K,
                     block_n, cvh::make_dropout(0.f, 0, 0), stream);
}

extern "C" int cv_gemm_bf16_dropout(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major,
                                    int64_t ldb, void* Cout, int c_is_f32, int64_t ldc, void* C2, const void* bias,
                                    int act, float* absmax, int M, int N, int K, int block_n, float dropout_p,
                                    uint64_t seed, uint32_t site, void* stream) {
    return gemm_impl(A, a_mn_major, lda, B, b_mn_major, ldb, Cout, c_is_f32, ldc, C2, bias, act, absmax, M, N, K,
                     block_n, cvh::make_dropout(dropout_p, seed, site), stream);
}
