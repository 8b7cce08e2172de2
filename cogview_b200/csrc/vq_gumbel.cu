// Gumbel-softmax quantiser of the VQ-VAE (vqvae/vqvae_zc.py, Quantize.forward_ with continuous_relax=True: soft
// :55-60, hard :61-65, the KL of :89-90, gumbel_softmax :284-346).
//
//   cv_gumbel_noise     the Gumbel(0, 1) noise g[row, code] the two kernels below use, written out (a test hook)
//   cv_vq_gumbel_fwd    per row of fp32 scores s = z.E: y = softmax((a + g) / tau) with a = 2 s - |e|^2, its arg-max,
//                       optionally the KL term of the noiseless softmax qy = softmax(a)
//   cv_vq_gumbel_bwd    da = y (dy - <y, dy>) / tau + c qy (log(qy K + 1e-20) + t - <qy, log(qy K + 1e-20) + t>),
//                       t = qy K / (qy K + 1e-20), and each row's sum of da
//
// |z|^2 of dist (:43-47) is the same for every code of a row, so it cancels in every softmax and arg-max here.
//
// Noise.  g = -log(-log(u)), u = (k + 1/2) 2^-23 from the top 23 bits k of a Philox4x32-10 word: u lies in
// [2^-24, 1 - 2^-24], both logarithms are finite, g lies in [-2.8, 16.7].  The four codes 4q .. 4q + 3 of a row take
// the four words of counter (row << 32 | q) under the caller's seed, so the noise is a function of (seed, absolute
// row, code) alone: independent of the grid and of how the caller splits the rows, and the backward regenerates it
// instead of storing it.
//
// One CTA of 256 threads per row; thread t owns the float4 groups t, t + 256, ...  Each pass re-reads the row's
// scores (L1/L2 hits after the first pass) and regenerates the noise.  Every reduction has a fixed order: per-thread
// in index order, then a fixed butterfly over the warp and warp 0 over the eight warp results, so equal inputs give
// equal bits.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

constexpr int GS_THREADS = 256;
constexpr int GS_WARPS = GS_THREADS / 32;
constexpr uint32_t GUMBEL_STREAM = 0x47554D42u;      // Philox stream id of the quantiser noise ("GUMB")

__device__ __forceinline__ float gumbel_of_word(uint32_t w) {
    const float u = ((float)(w >> 9) + 0.5f) * 1.1920928955078125e-07f;    // (2k + 1) 2^-24, exact in fp32
    return -logf(-logf(u));
}

__device__ __forceinline__ float4 gumbel4(uint64_t seed, int64_t row, int q) {
    const uint4 r = philox4x32_10(seed, ((uint64_t)row << 32) | (uint32_t)q, GUMBEL_STREAM);
    return make_float4(gumbel_of_word(r.x), gumbel_of_word(r.y), gumbel_of_word(r.z), gumbel_of_word(r.w));
}

__device__ __forceinline__ float f4(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

// online softmax state: running max m, sum S of exp(x - m) and sum T of exp(x - m) d; an empty state (S = 0,
// m = -inf) contributes nothing to a merge
struct Soft { float m, S, T; };

__device__ __forceinline__ void soft_add(Soft& s, float x, float d) {
    if (x > s.m) {
        const float r = s.S == 0.f ? 0.f : expf(s.m - x);
        s.S = s.S * r + 1.f;
        s.T = s.T * r + d;
        s.m = x;
    } else {
        const float e = expf(x - s.m);
        s.S += e;
        s.T += e * d;
    }
}
__device__ __forceinline__ Soft soft_merge(const Soft& a, const Soft& b) {
    const float M = fmaxf(a.m, b.m);
    const float ra = a.S == 0.f ? 0.f : expf(a.m - M), rb = b.S == 0.f ? 0.f : expf(b.m - M);
    return Soft{M, a.S * ra + b.S * rb, a.T * ra + b.T * rb};
}
__device__ __forceinline__ Soft soft_shfl(const Soft& s, int o) {
    return Soft{__shfl_xor_sync(0xffffffffu, s.m, o), __shfl_xor_sync(0xffffffffu, s.S, o),
                __shfl_xor_sync(0xffffffffu, s.T, o)};
}

// arg-max: larger value wins, the lower index on equal values
__device__ __forceinline__ void best_take(float& v, int& i, float v2, int i2) {
    if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

// block-wide reductions in a fixed order; every thread gets the result
struct RowRed {
    Soft soft[2][GS_WARPS];
    float val[GS_WARPS];
    int idx[GS_WARPS];
    float sum[GS_WARPS];
};

__device__ __forceinline__ Soft block_soft(Soft s, Soft* sh) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = soft_merge(s, soft_shfl(s, o));
    if (lane == 0) sh[warp] = s;
    __syncthreads();
    Soft t = sh[0];
#pragma unroll
    for (int w = 1; w < GS_WARPS; ++w) t = soft_merge(t, sh[w]);
    return t;
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    v = warp_sum(v);
    __syncthreads();                                   // sh may still be read from an earlier call
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < GS_WARPS; ++w) t += sh[w];
    return t;
}

__device__ __forceinline__ int block_argmax(float v, int i, RowRed& red) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        best_take(v, i, __shfl_xor_sync(0xffffffffu, v, o), __shfl_xor_sync(0xffffffffu, i, o));
    if (lane == 0) { red.val[warp] = v; red.idx[warp] = i; }
    __syncthreads();
    float bv = red.val[0];
    int bi = red.idx[0];
#pragma unroll
    for (int w = 1; w < GS_WARPS; ++w) best_take(bv, bi, red.val[w], red.idx[w]);
    return bi;
}

struct GumbelArgs {
    const float* s;          // [rows, ld] scores z.E
    int64_t ld;
    const float* e2;         // [K] |e|^2
    int K;
    uint64_t seed;
    int64_t row0;            // absolute index of row 0 (the noise counter)
    float inv_tau;
};

// log(qy K + 1e-20) + qy K / (qy K + 1e-20): d/dqy of qy log(qy K + 1e-20)
__device__ __forceinline__ float kl_g(float qy, float K) {
    const float t = qy * K + 1e-20f;
    return logf(t) + qy * K / t;
}

template <typename YT>
__device__ __forceinline__ void store4(YT* p, float a, float b, float c, float d);
template <>
__device__ __forceinline__ void store4<float>(float* p, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
template <>
__device__ __forceinline__ void store4<__nv_bfloat16>(__nv_bfloat16* p, float a, float b, float c, float d) {
    *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16x2(a, b), pack_bf16x2(c, d));
}

template <typename YT>
__global__ void __launch_bounds__(GS_THREADS)
vq_gumbel_fwd_kernel(const GumbelArgs p, YT* __restrict__ y, int64_t ldy, int64_t* __restrict__ idx_out,
                     float* __restrict__ kl_out) {
    __shared__ RowRed red;
    const int64_t row = blockIdx.x;
    const int64_t arow = p.row0 + row;
    const float* s = p.s + row * p.ld;
    const int G = p.K / 4;
    const bool want_kl = kl_out != nullptr;

    // pass 1: the noised softmax state and arg-max; the noiseless softmax state for the KL
    Soft sv{-INFINITY, 0.f, 0.f}, sa{-INFINITY, 0.f, 0.f};
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int q = threadIdx.x; q < G; q += GS_THREADS) {
        const float4 sc = *reinterpret_cast<const float4*>(s + 4 * q);
        const float4 ee = *reinterpret_cast<const float4*>(p.e2 + 4 * q);
        const float4 g = gumbel4(p.seed, arow, q);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float a = 2.f * f4(sc, e) - f4(ee, e);
            const float v = (a + f4(g, e)) * p.inv_tau;
            soft_add(sv, v, 0.f);
            if (want_kl) soft_add(sa, a, 0.f);
            if (v > bv) { bv = v; bi = 4 * q + e; }     // index order within the thread: the first maximum
        }
    }
    const int best = block_argmax(bv, bi, red);
    const Soft tv = block_soft(sv, red.soft[0]);
    const float inv_S = 1.f / tv.S;
    if (threadIdx.x == 0 && idx_out != nullptr) idx_out[row] = best;

    if (want_kl) {   // pass 2: sum_j qy_j log(qy_j K + 1e-20)
        const Soft ta = block_soft(sa, red.soft[1]);
        const float inv_Sa = 1.f / ta.S, Kf = (float)p.K;
        float acc = 0.f;
        for (int q = threadIdx.x; q < G; q += GS_THREADS) {
            const float4 sc = *reinterpret_cast<const float4*>(s + 4 * q);
            const float4 ee = *reinterpret_cast<const float4*>(p.e2 + 4 * q);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float qy = expf(2.f * f4(sc, e) - f4(ee, e) - ta.m) * inv_Sa;
                acc += qy * logf(qy * Kf + 1e-20f);
            }
        }
        const float kl = block_sum(acc, red.sum);
        if (threadIdx.x == 0) kl_out[row] = kl;
    }

    if (y != nullptr) {   // pass 3: y
        YT* yr = y + row * ldy;
        for (int q = threadIdx.x; q < G; q += GS_THREADS) {
            const float4 sc = *reinterpret_cast<const float4*>(s + 4 * q);
            const float4 ee = *reinterpret_cast<const float4*>(p.e2 + 4 * q);
            const float4 g = gumbel4(p.seed, arow, q);
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) o[e] = expf(((2.f * f4(sc, e) - f4(ee, e)) + f4(g, e)) * p.inv_tau - tv.m) * inv_S;
            store4<YT>(yr + 4 * q, o[0], o[1], o[2], o[3]);
        }
    }
}

__global__ void __launch_bounds__(GS_THREADS)
vq_gumbel_bwd_kernel(const GumbelArgs p, const float* __restrict__ dy, int64_t lddy, float kl_scale,
                     __nv_bfloat16* __restrict__ da, int64_t ldda, float* __restrict__ rowsum) {
    __shared__ RowRed red;
    const int64_t row = blockIdx.x;
    const int64_t arow = p.row0 + row;
    const float* s = p.s + row * p.ld;
    const float* d = dy != nullptr ? dy + row * lddy : nullptr;
    const int G = p.K / 4;
    const bool want_y = dy != nullptr, want_kl = kl_scale != 0.f;
    const float Kf = (float)p.K;

    // pass 1: softmax states of v = (a + g) / tau (with sum_j exp(v_j - m) dy_j) and of a
    Soft sv{-INFINITY, 0.f, 0.f}, sa{-INFINITY, 0.f, 0.f};
    for (int q = threadIdx.x; q < G; q += GS_THREADS) {
        const float4 sc = *reinterpret_cast<const float4*>(s + 4 * q);
        const float4 ee = *reinterpret_cast<const float4*>(p.e2 + 4 * q);
        if (want_y) {
            const float4 dd = *reinterpret_cast<const float4*>(d + 4 * q);
            const float4 g = gumbel4(p.seed, arow, q);
#pragma unroll
            for (int e = 0; e < 4; ++e)
                soft_add(sv, ((2.f * f4(sc, e) - f4(ee, e)) + f4(g, e)) * p.inv_tau, f4(dd, e));
        }
        if (want_kl) {
#pragma unroll
            for (int e = 0; e < 4; ++e) soft_add(sa, 2.f * f4(sc, e) - f4(ee, e), 0.f);
        }
    }
    const Soft tv = block_soft(sv, red.soft[0]);
    const Soft ta = block_soft(sa, red.soft[1]);
    const float inv_S = 1.f / tv.S, ydy = tv.T / tv.S;
    const float inv_Sa = 1.f / ta.S;

    float qg = 0.f;        // <qy, log(qy K + 1e-20) + t>
    if (want_kl) {         // pass 2
        float acc = 0.f;
        for (int q = threadIdx.x; q < G; q += GS_THREADS) {
            const float4 sc = *reinterpret_cast<const float4*>(s + 4 * q);
            const float4 ee = *reinterpret_cast<const float4*>(p.e2 + 4 * q);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float qy = expf(2.f * f4(sc, e) - f4(ee, e) - ta.m) * inv_Sa;
                acc += qy * kl_g(qy, Kf);
            }
        }
        qg = block_sum(acc, red.sum);
    }

    // pass 3: da and its row sum
    __nv_bfloat16* dar = da + row * ldda;
    float rs = 0.f;
    for (int q = threadIdx.x; q < G; q += GS_THREADS) {
        const float4 sc = *reinterpret_cast<const float4*>(s + 4 * q);
        const float4 ee = *reinterpret_cast<const float4*>(p.e2 + 4 * q);
        float o[4] = {0.f, 0.f, 0.f, 0.f};
        if (want_y) {
            const float4 dd = *reinterpret_cast<const float4*>(d + 4 * q);
            const float4 g = gumbel4(p.seed, arow, q);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float yv = expf(((2.f * f4(sc, e) - f4(ee, e)) + f4(g, e)) * p.inv_tau - tv.m) * inv_S;
                o[e] = yv * (f4(dd, e) - ydy) * p.inv_tau;
            }
        }
        if (want_kl) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float qy = expf(2.f * f4(sc, e) - f4(ee, e) - ta.m) * inv_Sa;
                o[e] += kl_scale * qy * (kl_g(qy, Kf) - qg);
            }
        }
        rs += (o[0] + o[1]) + (o[2] + o[3]);
        store4<__nv_bfloat16>(dar + 4 * q, o[0], o[1], o[2], o[3]);
    }
    const float total = block_sum(rs, red.sum);
    if (threadIdx.x == 0) rowsum[row] = total;
}

__global__ void gumbel_noise_kernel(uint64_t seed, int64_t row0, int64_t rows, int K, float* __restrict__ out) {
    const int G = K / 4;
    const int64_t n = rows * G;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / G;
        const int q = (int)(i - r * G);
        *reinterpret_cast<float4*>(out + r * K + 4 * q) = gumbel4(seed, row0 + r, q);
    }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int cv_gumbel_noise(uint64_t seed, int64_t row0, int64_t rows, int K, float* out, void* stream) {
    CV_REQUIRE(out != nullptr && aligned16(out), "out must be a 16-byte aligned pointer");
    CV_REQUIRE(rows > 0 && row0 >= 0 && K > 0 && K % 4 == 0, "rows and K must be positive, K a multiple of 4");
    CV_REQUIRE(row0 + rows <= (int64_t)1 << 32, "row indices must fit in 32 bits");
    const int64_t n = rows * (K / 4);
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)cvh::num_sms() * 16) blocks = (int64_t)cvh::num_sms() * 16;
    gumbel_noise_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(seed, row0, rows, K, out);
    CV_LAUNCH_CHECK();
    return 0;
}

static int check_common(const float* s, int64_t ld, const float* e2, int64_t rows, int K, int64_t row0, float tau) {
    CV_REQUIRE(s && e2, "null pointer");
    CV_REQUIRE(rows > 0 && rows < ((int64_t)1 << 31) && row0 >= 0 && row0 + rows <= (int64_t)1 << 32,
               "rows must be positive and row indices fit in 32 bits");
    CV_REQUIRE(K > 0 && K % 4 == 0 && ld >= K && ld % 4 == 0, "K and ld must be multiples of 4, ld >= K");
    CV_REQUIRE(aligned16(s) && aligned16(e2), "s and e2 must be 16-byte aligned");
    CV_REQUIRE(tau > 0.f && isfinite(tau), "temperature must be positive and finite");
    return 0;
}

extern "C" int cv_vq_gumbel_fwd(const float* s, int64_t ld, const float* e2, int64_t rows, int K, uint64_t seed,
                                int64_t row0, float tau, void* y, int y_f32, int64_t ldy, int64_t* idx, float* kl,
                                void* stream) {
    const int rc = check_common(s, ld, e2, rows, K, row0, tau);
    if (rc != 0) return rc;
    CV_REQUIRE(y || idx || kl, "nothing to compute");
    CV_REQUIRE(y == nullptr || (ldy >= K && ldy % (y_f32 ? 4 : 8) == 0 && aligned16(y)),
               "y rows must be 16-byte aligned with ldy >= K");
    GumbelArgs p{s, ld, e2, K, seed, row0, 1.f / tau};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (y_f32)
        vq_gumbel_fwd_kernel<float><<<(unsigned)rows, GS_THREADS, 0, st>>>(p, static_cast<float*>(y), ldy, idx, kl);
    else
        vq_gumbel_fwd_kernel<__nv_bfloat16><<<(unsigned)rows, GS_THREADS, 0, st>>>(
            p, static_cast<__nv_bfloat16*>(y), ldy, idx, kl);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_vq_gumbel_bwd(const float* s, int64_t ld, const float* e2, int64_t rows, int K, uint64_t seed,
                                int64_t row0, float tau, const float* dy, int64_t lddy, float kl_scale, void* da,
                                int64_t ldda, float* rowsum, void* stream) {
    const int rc = check_common(s, ld, e2, rows, K, row0, tau);
    if (rc != 0) return rc;
    CV_REQUIRE(da && rowsum, "null pointer");
    CV_REQUIRE(dy != nullptr || kl_scale != 0.f, "nothing to differentiate: no dy and no KL term");
    CV_REQUIRE(dy == nullptr || (lddy >= K && lddy % 4 == 0 && aligned16(dy)), "dy rows must be 16-byte aligned");
    CV_REQUIRE(ldda >= K && ldda % 8 == 0 && aligned16(da), "da rows must be 16-byte aligned with ldda >= K");
    CV_REQUIRE(isfinite(kl_scale), "kl_scale must be finite");
    GumbelArgs p{s, ld, e2, K, seed, row0, 1.f / tau};
    vq_gumbel_bwd_kernel<<<(unsigned)rows, GS_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        p, dy, lddy, kl_scale, static_cast<__nv_bfloat16*>(da), ldda, rowsum);
    CV_LAUNCH_CHECK();
    return 0;
}
