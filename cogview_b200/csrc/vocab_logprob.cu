// cv_vocab_logprob: logp[m] = logit(m, target[m]) - logsumexp_{v in [v_begin, v_end)} logit(m, v), with
// logit(m, v) = H[m, :] . W[v, :] — the caption log-likelihood of post-selection (generation/sampling.py:214-230:
// logits of every position, -inf on the image vocabulary, log(softmax), gather) for the scored rows only, without
// writing a logit to global memory.
//
// Design (sm_90a):
//   vocab_lse_kernel   the persistent wgmma GEMM of csrc/gemm.cu (its TMA ring and main loop, gemm_ring.cuh) over
//                      H [M, K] and the window's rows of W, 128 x 256 tiles.  The epilogue works on the fp32
//                      accumulators in registers: per row the tile's max and sum of exp(x - max) over the columns
//                      inside the window (masked by column index: a zero-filled column beyond the window would be a
//                      logit of 0, not an absent one), reduced over the four threads that share a row by shuffles,
//                      one (max, sum) pair per (column tile, row).  The tile holding target[m] writes that logit.
//                      Tiles are numbered row tile fastest, so the CTAs running at any moment all work on a few
//                      consecutive slabs of W: every row tile of a slab reads it while it is in L2, and W is read
//                      from HBM about once per call, not once per row tile.
//   vocab_lse_combine  one thread per row folds the row's pairs in column-tile order (a fixed order: equal inputs,
//                      equal bits) and subtracts the log-sum-exp from the target logit.
//
// The training loss over the whole vocabulary without logits (model/gpt2_modeling.py _VocabXentFn):
//   cv_vocab_xent_fwd      vocab_lse_kernel over [0, V), then vocab_xent_combine: the same fold, writing the
//                          per-token loss lse - logit(target) and the row's lse for the backward.
//   cv_vocab_xent_dlogits  vocab_xent_dlogits_kernel recomputes the logits of a column window [v_begin, v_end) on the
//                          same ring, main loop and tile order, and its epilogue turns the fp32 accumulators into
//                          grad * (exp(logit - lse) - [v == target]), stored as bf16 straight from registers.
#include <math.h>

#include "common.cuh"
#include "gemm_ring.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {

using namespace cv;
using namespace cv::ring;

constexpr int VBN = 256;

struct VlpParams {
    int M, n_win;                  // rows; window width v_end - v_begin (columns 0 .. n_win - 1 of the W tensor map)
    int num_m_blocks, num_tiles, num_k_blocks;
    const int64_t* target;         // [M] absolute vocabulary ids
    int v_begin;
    float2* part;                  // [column tiles, M]: (max, sum exp(x - max)) of the row over the tile's columns
    float* tlogit;                 // [M]: logit of the target (written only when it lies in the window)
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
vocab_lse_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW, const VlpParams p) {
    extern __shared__ uint8_t smem_raw[];
    const Ring<VBN> ring(smem_raw);
    const int wg = threadIdx.x >> 7;
    const int tid = threadIdx.x & 127;

    if (threadIdx.x == 0) ring.init(&tmH, &tmW);
    __syncthreads();

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tid == 0) {
            RingPos pos;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x)
                load_tile<VBN, false, false>(ring, pos, &tmH, &tmW, (tile % p.num_m_blocks) * BM,
                                             (tile / p.num_m_blocks) * VBN, VBN, p.num_k_blocks);
        }
        return;
    }
    setmaxnreg_inc<232>();
    const int half = wg - 1;
    const int warp = tid >> 5, lane = tid & 31;
    const int r_in = 64 * half + 16 * warp + (lane >> 2);   // this thread's rows: r_in and r_in + 8
    const int c_in = 2 * (lane & 3);                        // and columns 8i + c_in, + 1
    RingPos pos;
    float acc[VBN / 2];
#pragma unroll
    for (int i = 0; i < VBN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int m0 = (tile % p.num_m_blocks) * BM, nt = tile / p.num_m_blocks, n0 = nt * VBN;
        mma_tile<VBN, false, false>(ring, pos, acc, half, lane, true, p.num_k_blocks);
        const int lim = p.n_win - n0 - c_in;                // column 8i + e of this thread is in the window iff < lim
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + r_in + 8 * h;
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < VBN / 8; ++i) {
                if (8 * i < lim) mx = fmaxf(mx, acc[4 * i + 2 * h]);
                if (8 * i + 1 < lim) mx = fmaxf(mx, acc[4 * i + 2 * h + 1]);
            }
            // the four lanes of a row hold all of the tile's columns, and the tile at least one column of the window
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < VBN / 8; ++i) {
                if (8 * i < lim) s += __expf(acc[4 * i + 2 * h] - mx);
                if (8 * i + 1 < lim) s += __expf(acc[4 * i + 2 * h + 1] - mx);
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            if (row < p.M) {
                if ((lane & 3) == 0) p.part[(size_t)nt * p.M + row] = make_float2(mx, s);
                const int64_t t = p.target[row] - p.v_begin - n0 - c_in;   // column 8i + e of this thread, if any
                if (t >= 0 && t < VBN && (t & 6) == 0) {
                    const int ti = (int)(t >> 3), te = (int)(t & 1);
                    float v = 0.f;
#pragma unroll
                    for (int i = 0; i < VBN / 8; ++i)
                        if (i == ti) v = te ? acc[4 * i + 2 * h + 1] : acc[4 * i + 2 * h];
                    if (t < lim) p.tlogit[row] = v;
                }
            }
        }
    }
}

__global__ void vocab_lse_combine(const float2* __restrict__ part, const float* __restrict__ tlogit,
                                  const int64_t* __restrict__ target, int M, int n_tiles, int v_begin, int v_end,
                                  float* __restrict__ logp) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    float mx = -INFINITY, s = 0.f;
    for (int t = 0; t < n_tiles; ++t) {
        const float2 q = part[(size_t)t * M + m];
        const float nm = fmaxf(mx, q.x);
        s = s * expf(mx - nm) + q.y * expf(q.x - nm);
        mx = nm;
    }
    const int64_t tg = target[m];
    logp[m] = (tg >= v_begin && tg < v_end) ? tlogit[m] - (mx + logf(s)) : -INFINITY;
}

// loss[m] = lse[m] - logit(m, target[m]), written in the logits route's rounding (ce_fwd_kernel, csrc/misc.cu:
// log(sum) - (logit - max)); NaN for a target outside [0, V).
__global__ void vocab_xent_combine(const float2* __restrict__ part, const float* __restrict__ tlogit,
                                   const int64_t* __restrict__ target, int M, int n_tiles, int V,
                                   float* __restrict__ loss, float* __restrict__ lse) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    float mx = -INFINITY, s = 0.f;
    for (int t = 0; t < n_tiles; ++t) {
        const float2 q = part[(size_t)t * M + m];
        const float nm = fmaxf(mx, q.x);
        s = s * expf(mx - nm) + q.y * expf(q.x - nm);
        mx = nm;
    }
    const int64_t tg = target[m];
    const float ls = logf(s);
    loss[m] = (tg >= 0 && tg < V) ? ls - (tlogit[m] - mx) : __int_as_float(0x7fc00000);
    lse[m] = mx + ls;
}

struct XentParams {
    int M, n_win;                  // rows; window width v_end - v_begin (columns 0 .. n_win - 1 of the W tensor map)
    int num_m_blocks, num_tiles, num_k_blocks;
    const int64_t* target;         // [M] absolute vocabulary ids
    int v_begin;
    const float* lse;              // [M] log-sum-exp of the row over the whole vocabulary (cv_vocab_xent_fwd)
    const float* grad;             // [M] dL / dloss[m]
    __nv_bfloat16* D;              // [M, ldd]: column v - v_begin
    int64_t ldd;
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
vocab_xent_dlogits_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW,
                          const XentParams p) {
    extern __shared__ uint8_t smem_raw[];
    const Ring<VBN> ring(smem_raw);
    const int wg = threadIdx.x >> 7;
    const int tid = threadIdx.x & 127;

    if (threadIdx.x == 0) ring.init(&tmH, &tmW);
    __syncthreads();

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tid == 0) {
            RingPos pos;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x)
                load_tile<VBN, false, false>(ring, pos, &tmH, &tmW, (tile % p.num_m_blocks) * BM,
                                             (tile / p.num_m_blocks) * VBN, VBN, p.num_k_blocks);
        }
        return;
    }
    setmaxnreg_inc<232>();
    const int half = wg - 1;
    const int warp = tid >> 5, lane = tid & 31;
    const int r_in = 64 * half + 16 * warp + (lane >> 2);   // this thread's rows: r_in and r_in + 8
    const int c_in = 2 * (lane & 3);                        // and columns 8i + c_in, + 1
    RingPos pos;
    float acc[VBN / 2];
#pragma unroll
    for (int i = 0; i < VBN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int m0 = (tile % p.num_m_blocks) * BM, n0 = (tile / p.num_m_blocks) * VBN;
        mma_tile<VBN, false, false>(ring, pos, acc, half, lane, true, p.num_k_blocks);
        const int lim = p.n_win - n0 - c_in;                // column 8i + e of this thread is in the window iff < lim
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + r_in + 8 * h;
            if (row >= p.M) continue;
            const float l = p.lse[row], g = p.grad[row];
            const int64_t t = p.target[row] - p.v_begin - n0 - c_in;   // the target's column 8i + e, if any
            __nv_bfloat16* d = p.D + (size_t)row * p.ldd + n0 + c_in;
#pragma unroll
            for (int i = 0; i < VBN / 8; ++i) {
                if (8 * i >= lim) continue;
                const float v0 = g * (__expf(acc[4 * i + 2 * h] - l) - (t == 8 * i ? 1.f : 0.f));
                const float v1 = g * (__expf(acc[4 * i + 2 * h + 1] - l) - (t == 8 * i + 1 ? 1.f : 0.f));
                if (8 * i + 1 < lim) *reinterpret_cast<uint32_t*>(d + 8 * i) = pack_bf16x2(v0, v1);
                else d[8 * i] = __float2bfloat16_rn(v0);
            }
        }
    }
}

int64_t col_tiles(int v_begin, int v_end) { return ((int64_t)v_end - v_begin + VBN - 1) / VBN; }

bool tiles_fit(int M, int v_begin, int v_end) {
    return col_tiles(v_begin, v_end) * ((M + BM - 1) / BM) < (1ll << 31);
}

// vocab_lse_kernel over the window [v_begin, v_end): part = workspace, tlogit after it (see VlpParams)
int launch_lse(const void* H, int64_t ldh, const void* W, int64_t ldw, const int64_t* target, float* workspace, int M,
               int K, int v_begin, int v_end, cudaStream_t s) {
    const int64_t n_tiles = col_tiles(v_begin, v_end);
    const int64_t m_blocks = (M + BM - 1) / BM;

    VlpParams p;
    p.M = M;
    p.n_win = v_end - v_begin;
    p.num_m_blocks = (int)m_blocks;
    p.num_tiles = (int)(n_tiles * m_blocks);
    p.num_k_blocks = (K + BK - 1) / BK;
    p.target = target;
    p.v_begin = v_begin;
    p.part = reinterpret_cast<float2*>(workspace);
    p.tlogit = workspace + 2 * n_tiles * M;

    alignas(64) CUtensorMap tmH, tmW;
    int rc = cvh::encode_tmap_2d_bf16(&tmH, H, M, K, ldh, BM, BK);
    if (rc) return rc;
    // the window's rows of W only: columns of the last tile beyond v_end are zero-filled and masked by index
    rc = cvh::encode_tmap_2d_bf16(&tmW, static_cast<const __nv_bfloat16*>(W) + (int64_t)v_begin * ldw, p.n_win, K,
                                  ldw, 128, BK);
    if (rc) return rc;

    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(vocab_lse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Cfg<VBN>::SMEM_BYTES));
        attr_set = true;
    }
    const int grid = p.num_tiles < cvh::gemm_sms() ? p.num_tiles : cvh::gemm_sms();
    vocab_lse_kernel<<<grid, NUM_THREADS, Cfg<VBN>::SMEM_BYTES, s>>>(tmH, tmW, p);
    CV_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int64_t cv_vocab_logprob_workspace_bytes(int M, int v_begin, int v_end) {
    if (M <= 0 || v_begin < 0 || v_end <= v_begin) return 0;
    return (col_tiles(v_begin, v_end) * 2 + 1) * (int64_t)M * (int64_t)sizeof(float);
}

extern "C" int cv_vocab_logprob(const void* H, int64_t ldh, const void* W, int64_t ldw, const int64_t* target,
                                float* logp, float* workspace, int M, int K, int v_begin, int v_end, void* stream) {
    CV_REQUIRE(H && W && target && logp && workspace, "null pointer");
    CV_REQUIRE(M > 0 && K > 0, "M and K must be positive");
    CV_REQUIRE(v_begin >= 0 && v_end > v_begin, "need 0 <= v_begin < v_end");
    CV_REQUIRE(ldh >= K && ldw >= K && ldh % 8 == 0 && ldw % 8 == 0,
               "ldh and ldw must be >= K and multiples of 8 elements (16-byte TMA strides)");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(H) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
               "H and W must be 16-byte aligned");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "workspace must be 8-byte aligned");
    CV_REQUIRE(tiles_fit(M, v_begin, v_end), "too many tiles");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int rc = launch_lse(H, ldh, W, ldw, target, workspace, M, K, v_begin, v_end, s);
    if (rc) return rc;
    const int n_tiles = (int)col_tiles(v_begin, v_end);
    vocab_lse_combine<<<(M + 127) / 128, 128, 0, s>>>(reinterpret_cast<const float2*>(workspace),
                                                      workspace + 2 * (int64_t)n_tiles * M, target, M, n_tiles,
                                                      v_begin, v_end, logp);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int64_t cv_vocab_xent_workspace_bytes(int M, int V) { return cv_vocab_logprob_workspace_bytes(M, 0, V); }

extern "C" int cv_vocab_xent_fwd(const void* H, int64_t ldh, const void* W, int64_t ldw, const int64_t* target,
                                 float* loss, float* lse, float* workspace, int M, int K, int V, void* stream) {
    CV_REQUIRE(H && W && target && loss && lse && workspace, "null pointer");
    CV_REQUIRE(M > 0 && K > 0 && V > 0, "M, K and V must be positive");
    CV_REQUIRE(ldh >= K && ldw >= K && ldh % 8 == 0 && ldw % 8 == 0,
               "ldh and ldw must be >= K and multiples of 8 elements (16-byte TMA strides)");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(H) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
               "H and W must be 16-byte aligned");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "workspace must be 8-byte aligned");
    CV_REQUIRE(tiles_fit(M, 0, V), "too many tiles");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int rc = launch_lse(H, ldh, W, ldw, target, workspace, M, K, 0, V, s);
    if (rc) return rc;
    const int n_tiles = (int)col_tiles(0, V);
    vocab_xent_combine<<<(M + 127) / 128, 128, 0, s>>>(reinterpret_cast<const float2*>(workspace),
                                                       workspace + 2 * (int64_t)n_tiles * M, target, M, n_tiles, V,
                                                       loss, lse);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_vocab_xent_dlogits(const void* H, int64_t ldh, const void* W, int64_t ldw, const int64_t* target,
                                     const float* lse, const float* grad_loss, void* D, int64_t ldd, int M, int K,
                                     int v_begin, int v_end, void* stream) {
    CV_REQUIRE(H && W && target && lse && grad_loss && D, "null pointer");
    CV_REQUIRE(M > 0 && K > 0, "M and K must be positive");
    CV_REQUIRE(v_begin >= 0 && v_end > v_begin, "need 0 <= v_begin < v_end");
    CV_REQUIRE(ldh >= K && ldw >= K && ldh % 8 == 0 && ldw % 8 == 0,
               "ldh and ldw must be >= K and multiples of 8 elements (16-byte TMA strides)");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(H) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
               "H and W must be 16-byte aligned");
    CV_REQUIRE(ldd >= (int64_t)v_end - v_begin && ldd % 2 == 0, "ldd must be >= v_end - v_begin and even");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(D) & 3) == 0, "D must be 4-byte aligned");
    CV_REQUIRE(tiles_fit(M, v_begin, v_end), "too many tiles");
    const int64_t n_tiles = col_tiles(v_begin, v_end);
    const int64_t m_blocks = (M + BM - 1) / BM;
    cudaStream_t s = static_cast<cudaStream_t>(stream);

    XentParams p;
    p.M = M;
    p.n_win = v_end - v_begin;
    p.num_m_blocks = (int)m_blocks;
    p.num_tiles = (int)(n_tiles * m_blocks);
    p.num_k_blocks = (K + BK - 1) / BK;
    p.target = target;
    p.v_begin = v_begin;
    p.lse = lse;
    p.grad = grad_loss;
    p.D = static_cast<__nv_bfloat16*>(D);
    p.ldd = ldd;

    alignas(64) CUtensorMap tmH, tmW;
    int rc = cvh::encode_tmap_2d_bf16(&tmH, H, M, K, ldh, BM, BK);
    if (rc) return rc;
    rc = cvh::encode_tmap_2d_bf16(&tmW, static_cast<const __nv_bfloat16*>(W) + (int64_t)v_begin * ldw, p.n_win, K,
                                  ldw, 128, BK);
    if (rc) return rc;

    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(vocab_xent_dlogits_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Cfg<VBN>::SMEM_BYTES));
        attr_set = true;
    }
    const int grid = p.num_tiles < cvh::gemm_sms() ? p.num_tiles : cvh::gemm_sms();
    vocab_xent_dlogits_kernel<<<grid, NUM_THREADS, Cfg<VBN>::SMEM_BYTES, s>>>(tmH, tmW, p);
    CV_LAUNCH_CHECK();
    return 0;
}
