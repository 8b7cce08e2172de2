// HBM-bound helper kernels of the transformer path: embedding gather / scatter, vocab cross-entropy,
// GELU backward, bias gradient (column sums), abs-max reduction.  All are coalesced, vectorised where the
// layout allows, and sized in multiples of the SM count.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

// ------------------------------------------------------------------------------------------------
// Embedding: hidden[r, :] = wte[ids[r], :] + wpe[pos[r], :]   (fp32 residual stream) + max|hidden|
//   VocabParallelEmbedding.forward  /root/reference/mpu/layers.py:117-133
//   + position embedding add        /root/reference/mpu/sparse_transformer.py:522-523
// ------------------------------------------------------------------------------------------------
__global__ void embed_fwd_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ pos,
                                 const __nv_bfloat16* __restrict__ wte, const __nv_bfloat16* __restrict__ wpe,
                                 float* __restrict__ out, float* __restrict__ absmax, int rows, int h,
                                 const DropoutArgs drop) {
    pdl_launch_dependents();   // lets a PDL-launched consumer (decode path) start its prologue early
    const int warps_per_block = blockDim.x >> 5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float mx = 0.f;
    for (int r = blockIdx.x * warps_per_block + warp; r < rows; r += gridDim.x * warps_per_block) {
        const __nv_bfloat16* a = wte + (size_t)ids[r] * h;
        const __nv_bfloat16* b = wpe + (size_t)pos[r] * h;
        float* o = out + (size_t)r * h;
        for (int i = lane * 8; i < h; i += 256) {
            uint4 ua = *reinterpret_cast<const uint4*>(a + i);
            uint4 ub = *reinterpret_cast<const uint4*>(b + i);
            const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&ua);
            const __nv_bfloat162* pb = reinterpret_cast<const __nv_bfloat162*>(&ub);
            float v[8];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                v[2 * t] = __low2float(pa[t]) + __low2float(pb[t]);
                v[2 * t + 1] = __high2float(pa[t]) + __high2float(pb[t]);
            }
            if (drop.p > 0.f) {   // embedding dropout (mpu/sparse_transformer.py:524)
                const uint64_t e = (uint64_t)r * h + i;
                dropout4(drop, e >> 2, v[0], v[1], v[2], v[3]);
                dropout4(drop, (e >> 2) + 1, v[4], v[5], v[6], v[7]);
            }
            *reinterpret_cast<float4*>(o + i) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(o + i + 4) = make_float4(v[4], v[5], v[6], v[7]);
#pragma unroll
            for (int t = 0; t < 8; ++t) mx = fmaxf(mx, fabsf(v[t]));
        }
    }
    if (absmax != nullptr) {
        mx = warp_max(mx);
        if (lane == 0 && mx > 0.f) atomic_max_nonneg(absmax, mx);
    }
}

// dwte[ids[r]] += dx[r], dwpe[pos[r]] += dx[r]  (bf16 gradients).  One warp per task = (table, row r); the task whose
// row is the first one carrying its index adds every row carrying that index, in row order, and the others do nothing.
// A token or position that occurs three or more times thus gets the same gradient bits on every run (atomics would add
// in arrival order).
__global__ void embed_bwd_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ pos,
                                 const float* __restrict__ dx, __nv_bfloat16* __restrict__ dwte,
                                 __nv_bfloat16* __restrict__ dwpe, int rows, int h, const DropoutArgs drop) {
    const int warps_per_block = blockDim.x >> 5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int task = blockIdx.x * warps_per_block + warp; task < 2 * rows; task += gridDim.x * warps_per_block) {
        const bool is_pos = task >= rows;
        const int r = is_pos ? task - rows : task;
        const int64_t* idx = is_pos ? pos : ids;
        const int64_t v = idx[r];
        bool seen = false;
        for (int j0 = 0; j0 < r && !seen; j0 += 32) seen = __any_sync(0xffffffffu, j0 + lane < r && idx[j0 + lane] == v);
        if (seen) continue;
        __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>((is_pos ? dwpe : dwte) + (size_t)v * h);
        for (int j0 = r; j0 < rows; j0 += 32) {
            unsigned m = __ballot_sync(0xffffffffu, j0 + lane < rows && idx[j0 + lane] == v);
            while (m) {
                const int j = j0 + __ffs(m) - 1;
                m &= m - 1;
                const float4* d = reinterpret_cast<const float4*>(dx + (size_t)j * h);
                for (int i = lane; i < h / 4; i += 32) {
                    float4 x = d[i];
                    if (drop.p > 0.f) dropout4(drop, ((uint64_t)j * h + 4 * (uint64_t)i) >> 2, x.x, x.y, x.z, x.w);
                    // dx is rounded to bf16 before the add, and the sum rounded again, as a bf16 atomicAdd does: a
                    // row that occurs once or twice gets exactly the bits it got from atomics
                    const float2 a = __bfloat1622float2(o[2 * i]), b = __bfloat1622float2(o[2 * i + 1]);
                    const float2 p = __bfloat1622float2(__floats2bfloat162_rn(x.x, x.y));
                    const float2 q = __bfloat1622float2(__floats2bfloat162_rn(x.z, x.w));
                    o[2 * i] = __floats2bfloat162_rn(a.x + p.x, a.y + p.y);
                    o[2 * i + 1] = __floats2bfloat162_rn(b.x + q.x, b.y + q.y);
                }
            }
        }
    }
}

__global__ void dropout_mask_kernel(uint8_t* __restrict__ out, size_t n, const DropoutArgs drop) {
    for (size_t i4 = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i4 * 4 < n; i4 += (size_t)gridDim.x * blockDim.x) {
        float a = 1.f, b = 1.f, c = 1.f, e = 1.f;
        dropout4(drop, i4, a, b, c, e);
        const float v[4] = {a, b, c, e};
        for (int t = 0; t < 4; ++t)
            if (i4 * 4 + t < n) out[i4 * 4 + t] = v[t] != 0.f;
    }
}

DropoutArgs to_dev(const cvh::HostDropout& hd) {
    DropoutArgs d;
    d.p = hd.p; d.scale = hd.scale; d.threshold = hd.threshold; d.stream = hd.stream; d.seed = hd.seed;
    return d;
}

// ------------------------------------------------------------------------------------------------
// Vocab cross-entropy  (/root/reference/mpu/cross_entropy.py:27-104 at model-parallel size 1)
//   loss[r] = log(sum_j exp(l[r,j] - max_r)) - (l[r,target] - max_r)
//   dl[r,j] = (exp(l[r,j] - max_r) / sum_r - [j == target]) * g[r]
// One CTA per row; fp32 logits; the row maximum and sum are saved for the backward.
// ------------------------------------------------------------------------------------------------
constexpr int CE_THREADS = 512;

__device__ __forceinline__ float block_reduce_max(float v, float* sh) {
    v = warp_max(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = (lane < (blockDim.x >> 5)) ? sh[lane] : -INFINITY;
        t = warp_max(t);
        if (lane == 0) sh[0] = t;
    }
    __syncthreads();
    float r = sh[0];
    __syncthreads();
    return r;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* sh) {
    v = warp_sum(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = (lane < (blockDim.x >> 5)) ? sh[lane] : 0.f;
        t = warp_sum(t);
        if (lane == 0) sh[0] = t;
    }
    __syncthreads();
    float r = sh[0];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(CE_THREADS)
ce_fwd_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ target,
              float* __restrict__ loss, float* __restrict__ row_max, float* __restrict__ row_sum, int V) {
    __shared__ float sh[32];
    const int r = blockIdx.x;
    const float* l = logits + (size_t)r * ld;
    float mx = -INFINITY;
    for (int i = threadIdx.x * 4; i < V; i += CE_THREADS * 4) {
        if (i + 3 < V) {
            float4 v = *reinterpret_cast<const float4*>(l + i);
            mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
        } else {
            for (int j = i; j < V; ++j) mx = fmaxf(mx, l[j]);
        }
    }
    mx = block_reduce_max(mx, sh);
    float s = 0.f;
    for (int i = threadIdx.x * 4; i < V; i += CE_THREADS * 4) {
        if (i + 3 < V) {
            float4 v = *reinterpret_cast<const float4*>(l + i);
            s += (__expf(v.x - mx) + __expf(v.y - mx)) + (__expf(v.z - mx) + __expf(v.w - mx));
        } else {
            for (int j = i; j < V; ++j) s += __expf(l[j] - mx);
        }
    }
    s = block_reduce_sum(s, sh);
    if (threadIdx.x == 0) {
        const float pred = l[target[r]] - mx;
        loss[r] = logf(s) - pred;
        row_max[r] = mx;
        row_sum[r] = s;
    }
}

__global__ void __launch_bounds__(CE_THREADS)
ce_bwd_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ target,
              const float* __restrict__ row_max, const float* __restrict__ row_sum, const float* __restrict__ g,
              __nv_bfloat16* __restrict__ dlogits, int64_t ldd, int V) {
    const int r = blockIdx.x;
    const float* l = logits + (size_t)r * ld;
    __nv_bfloat16* d = dlogits + (size_t)r * ldd;
    const float mx = row_max[r], inv = 1.0f / row_sum[r], gr = g[r];
    const int tgt = (int)target[r];
    for (int i = threadIdx.x * 4; i < V; i += CE_THREADS * 4) {
        if (i + 3 < V) {
            float4 v = *reinterpret_cast<const float4*>(l + i);
            float o0 = __expf(v.x - mx) * inv, o1 = __expf(v.y - mx) * inv, o2 = __expf(v.z - mx) * inv,
                  o3 = __expf(v.w - mx) * inv;
            if (tgt == i) o0 -= 1.f;
            if (tgt == i + 1) o1 -= 1.f;
            if (tgt == i + 2) o2 -= 1.f;
            if (tgt == i + 3) o3 -= 1.f;
            uint2 u;
            u.x = pack_bf16x2(o0 * gr, o1 * gr);
            u.y = pack_bf16x2(o2 * gr, o3 * gr);
            *reinterpret_cast<uint2*>(d + i) = u;
        } else {
            for (int j = i; j < V; ++j) {
                float o = __expf(l[j] - mx) * inv - (j == tgt ? 1.f : 0.f);
                d[j] = __float2bfloat16_rn(o * gr);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// GELU backward: dpre = dact * gelu'(pre)   (bf16 in/out)   mpu/sparse_transformer.py:172-176
// ------------------------------------------------------------------------------------------------
__global__ void gelu_bwd_kernel(const __nv_bfloat16* __restrict__ pre, const __nv_bfloat16* __restrict__ dact,
                                __nv_bfloat16* __restrict__ dpre, size_t n8) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
        uint4 up = reinterpret_cast<const uint4*>(pre)[i];
        uint4 ud = reinterpret_cast<const uint4*>(dact)[i];
        const __nv_bfloat162* pp = reinterpret_cast<const __nv_bfloat162*>(&up);
        const __nv_bfloat162* pd = reinterpret_cast<const __nv_bfloat162*>(&ud);
        uint4 o;
        uint32_t* po = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            float a = gelu_tanh_grad(__low2float(pp[t])) * __low2float(pd[t]);
            float b = gelu_tanh_grad(__high2float(pp[t])) * __high2float(pd[t]);
            po[t] = pack_bf16x2(a, b);
        }
        reinterpret_cast<uint4*>(dpre)[i] = o;
    }
}

// ------------------------------------------------------------------------------------------------
// Column sums: db[c] = sum_r dy[r, c]   (bias gradients of the four linears)
// ------------------------------------------------------------------------------------------------
constexpr int COLSUM_SPLITS = 32;
__global__ void __launch_bounds__(128)
colsum_partial_kernel(const __nv_bfloat16* __restrict__ dy, int64_t ld, float* __restrict__ partials, int rows,
                      int cols) {
    // each thread owns two adjacent columns (bf16x2 loads, 256 B per warp row segment)
    const int c = (blockIdx.x * 128 + threadIdx.x) * 2;
    const int rows_per = (rows + gridDim.y - 1) / gridDim.y;
    const int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
    if (c >= cols) return;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 4
    for (int r = r0; r < r1; ++r) {
        __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(dy + (size_t)r * ld + c);
        s0 += __low2float(v);
        s1 += __high2float(v);
    }
    partials[(size_t)blockIdx.y * cols + c] = s0;
    partials[(size_t)blockIdx.y * cols + c + 1] = s1;
}
__global__ void colsum_finalize_kernel(const float* __restrict__ partials, int nparts, int cols,
                                       __nv_bfloat16* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float s = 0.f;
    for (int p = 0; p < nparts; ++p) s += partials[(size_t)p * cols + c];
    out[c] = __float2bfloat16_rn(s);
}

// ------------------------------------------------------------------------------------------------
// max|x| of a whole tensor (for LayerNorm inputs not produced by one of our kernels)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void absmax_kernel(const T* __restrict__ x, size_t n, float* __restrict__ out) {
    float mx = 0.f;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        mx = fmaxf(mx, fabsf((float)x[i]));
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0 && mx > 0.f) atomic_max_nonneg(out, mx);
}

int grid_for(size_t work_items, int threads) {
    size_t blocks = (work_items + threads - 1) / threads;
    size_t cap = (size_t)cvh::num_sms() * 8;
    return (int)(blocks < cap ? (blocks ? blocks : 1) : cap);
}

}  // namespace

extern "C" int cv_dropout_mask(uint8_t* out, int64_t n, float p, uint64_t seed, uint32_t site, void* stream) {
    CV_REQUIRE(out && n > 0 && p >= 0.f && p < 1.f, "bad argument");
    dropout_mask_kernel<<<grid_for((size_t)(n + 3) / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        out, (size_t)n, to_dev(cvh::make_dropout(p, seed, site)));
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_embed_fwd(const int64_t* ids, const int64_t* pos, const void* wte, const void* wpe, float* out,
                            float* absmax, int rows, int hidden, float dropout_p, uint64_t seed, uint32_t site,
                            void* stream) {
    CV_REQUIRE(ids && pos && wte && wpe && out, "null pointer");
    CV_REQUIRE(rows > 0 && hidden > 0 && hidden % 8 == 0, "hidden must be a multiple of 8");
    const int wpb = 8;
    int blocks = (rows + wpb - 1) / wpb;
    int cap = cvh::num_sms() * 4;
    embed_fwd_kernel<<<blocks < cap ? blocks : cap, wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(
        ids, pos, static_cast<const __nv_bfloat16*>(wte), static_cast<const __nv_bfloat16*>(wpe), out, absmax, rows,
        hidden, to_dev(cvh::make_dropout(dropout_p, seed, site)));
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_embed_bwd(const int64_t* ids, const int64_t* pos, const float* dx, void* dwte, void* dwpe, int rows,
                            int hidden, float dropout_p, uint64_t seed, uint32_t site, void* stream) {
    CV_REQUIRE(ids && pos && dx && dwte && dwpe, "null pointer");
    CV_REQUIRE(rows > 0 && hidden > 0 && hidden % 4 == 0, "hidden must be a multiple of 4");
    const int wpb = 8;
    int blocks = (2 * rows + wpb - 1) / wpb;
    int cap = cvh::num_sms() * 4;
    embed_bwd_kernel<<<blocks < cap ? blocks : cap, wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(
        ids, pos, dx, static_cast<__nv_bfloat16*>(dwte), static_cast<__nv_bfloat16*>(dwpe), rows, hidden,
        to_dev(cvh::make_dropout(dropout_p, seed, site)));
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_cross_entropy_fwd(const float* logits, int64_t ld, const int64_t* target, float* loss,
                                    float* row_max, float* row_sum, int rows, int vocab, void* stream) {
    CV_REQUIRE(logits && target && loss && row_max && row_sum, "null pointer");
    CV_REQUIRE(rows > 0 && vocab > 0 && ld % 4 == 0, "ld must be a multiple of 4");
    ce_fwd_kernel<<<rows, CE_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(logits, ld, target, loss, row_max,
                                                                            row_sum, vocab);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_cross_entropy_bwd(const float* logits, int64_t ld, const int64_t* target, const float* row_max,
                                    const float* row_sum, const float* grad_loss, void* dlogits, int64_t ldd, int rows,
                                    int vocab, void* stream) {
    CV_REQUIRE(logits && target && row_max && row_sum && grad_loss && dlogits, "null pointer");
    CV_REQUIRE(rows > 0 && vocab > 0 && ld % 4 == 0 && ldd % 4 == 0, "ld/ldd must be multiples of 4");
    ce_bwd_kernel<<<rows, CE_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        logits, ld, target, row_max, row_sum, grad_loss, static_cast<__nv_bfloat16*>(dlogits), ldd, vocab);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_gelu_bwd(const void* pre, const void* dact, void* dpre, int64_t n, void* stream) {
    CV_REQUIRE(pre && dact && dpre, "null pointer");
    CV_REQUIRE(n > 0 && n % 8 == 0, "element count must be a multiple of 8");
    const size_t n8 = (size_t)n / 8;
    gelu_bwd_kernel<<<grid_for(n8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(pre), static_cast<const __nv_bfloat16*>(dact),
        static_cast<__nv_bfloat16*>(dpre), n8);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int64_t cv_colsum_workspace_bytes(int cols) { return (int64_t)COLSUM_SPLITS * cols * sizeof(float); }

extern "C" int cv_colsum_bf16(const void* dy, int64_t ld, void* out, float* workspace, int rows, int cols,
                              void* stream) {
    CV_REQUIRE(dy && out && workspace, "null pointer");
    CV_REQUIRE(rows > 0 && cols > 0 && cols % 2 == 0 && ld % 2 == 0, "cols and ld must be even");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int splits = rows < COLSUM_SPLITS ? rows : COLSUM_SPLITS;
    dim3 grid((cols / 2 + 127) / 128, splits);
    colsum_partial_kernel<<<grid, 128, 0, s>>>(static_cast<const __nv_bfloat16*>(dy), ld, workspace, rows, cols);
    CV_LAUNCH_CHECK();
    colsum_finalize_kernel<<<(cols + 255) / 256, 256, 0, s>>>(workspace, splits, cols,
                                                             static_cast<__nv_bfloat16*>(out));
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_absmax(const void* x, int x_is_bf16, int64_t n, float* out, void* stream) {
    CV_REQUIRE(x && out && n > 0, "bad argument");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (x_is_bf16)
        absmax_kernel<<<grid_for((size_t)n, 256), 256, 0, s>>>(static_cast<const __nv_bfloat16*>(x), (size_t)n, out);
    else
        absmax_kernel<<<grid_for((size_t)n, 256), 256, 0, s>>>(static_cast<const float*>(x), (size_t)n, out);
    CV_LAUNCH_CHECK();
    return 0;
}
