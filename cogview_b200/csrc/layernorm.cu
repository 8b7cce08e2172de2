// Abs-max pre-scaled LayerNorm (the reference's `LayerNorm`, /root/reference/mpu/sparse_transformer.py:40-44):
//     y = FusedLayerNorm(x / (max|x| / 8)),   max over the WHOLE tensor, detached
// which is algebraically LN with a data-dependent epsilon:  (x - mu) / sqrt(var + eps * c^2) * gamma + beta,
// c = max|x| / 8.  The scalar max|x| is produced by whichever kernel wrote x (GEMM epilogue, the
// residual-adding variant of this kernel, or the embedding kernel) via atomicMax, so no extra pass over x.
//
// Sandwich-LN fusion (mpu/sparse_transformer.py:314-342): the `third`/`fourth` LayerNorms are applied to a
// bf16 GEMM output and immediately added to the fp32 residual stream; that variant (RES) also emits
// max|residual_out| for the LayerNorm that follows.
//
// HBM-bound: one warp per row, the row is staged once in shared memory (fp32) and re-read from there.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

constexpr int WARPS = 8;

__device__ __forceinline__ float ld_as_float(const float* p, size_t i) { return p[i]; }
__device__ __forceinline__ float ld_as_float(const __nv_bfloat16* p, size_t i) { return __bfloat162float(p[i]); }

// vector loads of 4 consecutive elements
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4(const __nv_bfloat16* p) {
    uint2 u = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&u.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&u.y);
    return make_float4(__low2float(a), __high2float(a), __low2float(b), __high2float(b));
}
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(__nv_bfloat16* p, float4 v) {
    uint2 u;
    u.x = pack_bf16x2(v.x, v.y);
    u.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(p) = u;
}
__device__ __forceinline__ float round_as(float v, const float*) { return v; }
__device__ __forceinline__ float round_as(float v, const __nv_bfloat16*) { return bf16_round(v); }

template <typename TIn, typename TOut, bool RES>
__global__ void __launch_bounds__(WARPS * 32)
ln_fwd_kernel(const TIn* __restrict__ x, const float* __restrict__ absmax_in, const __nv_bfloat16* __restrict__ gamma,
              const __nv_bfloat16* __restrict__ beta, float eps, const float* __restrict__ residual,
              TOut* __restrict__ out, float* __restrict__ absmax_out, float* __restrict__ mean_out,
              float* __restrict__ rstd_out, int rows, int cols) {
    extern __shared__ float srow_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* srow = srow_all + warp * cols;
    const float c = *absmax_in * 0.125f;
    const float eps_eff = eps * c * c;
    const float inv_n = 1.0f / cols;
    float omax = 0.f;
    for (int row = blockIdx.x * WARPS + warp; row < rows; row += gridDim.x * WARPS) {
        const TIn* xr = x + (size_t)row * cols;
        float s = 0.f;
        for (int i = lane * 4; i < cols; i += 128) {
            float4 v = ld4(xr + i);
            st4(srow + i, v);
            s += (v.x + v.y) + (v.z + v.w);
        }
        const float mean = warp_sum(s) * inv_n;
        float ss = 0.f;
        for (int i = lane * 4; i < cols; i += 128) {
            float4 v = ld4(srow + i);
            float a = v.x - mean, b = v.y - mean, d = v.z - mean, e = v.w - mean;
            ss += (a * a + b * b) + (d * d + e * e);
        }
        const float var = warp_sum(ss) * inv_n;
        const float rstd = rsqrtf(var + eps_eff);
        if (lane == 0 && mean_out != nullptr) {
            mean_out[row] = mean;
            rstd_out[row] = rstd;
        }
        TOut* orow = out + (size_t)row * cols;
        for (int i = lane * 4; i < cols; i += 128) {
            float4 v = ld4(srow + i);
            float4 g = ld4(gamma + i), bt = ld4(beta + i);
            float4 y;
            y.x = (v.x - mean) * rstd * g.x + bt.x;
            y.y = (v.y - mean) * rstd * g.y + bt.y;
            y.z = (v.z - mean) * rstd * g.z + bt.z;
            y.w = (v.w - mean) * rstd * g.w + bt.w;
            if (RES) {
                float4 r = ld4(residual + (size_t)row * cols + i);
                y.x += r.x; y.y += r.y; y.z += r.z; y.w += r.w;
            }
            st4(orow + i, y);
            if (absmax_out != nullptr) {
                omax = fmaxf(omax, fmaxf(fmaxf(fabsf(round_as(y.x, orow)), fabsf(round_as(y.y, orow))),
                                         fmaxf(fabsf(round_as(y.z, orow)), fabsf(round_as(y.w, orow)))));
            }
        }
        __syncwarp();
    }
    if (absmax_out != nullptr) {
        omax = warp_max(omax);
        if (lane == 0 && omax > 0.f) atomic_max_nonneg(absmax_out, omax);
    }
}

// Same operation with the row held in REGISTERS (cols <= 128 * NV): a lane issues all NV 16-byte loads of its row
// before the first use, so 16 resident warps keep ~160 KB in flight per SM — the shared-memory staged kernel above has
// only a few loads in flight per warp.
template <typename TIn, typename TOut, bool RES, int NV>
__global__ void __launch_bounds__(WARPS * 32, 2)
ln_fwd_reg_kernel(const TIn* __restrict__ x, const float* __restrict__ absmax_in, const __nv_bfloat16* __restrict__ gamma,
                  const __nv_bfloat16* __restrict__ beta, float eps, const float* __restrict__ residual,
                  TOut* __restrict__ out, float* __restrict__ absmax_out, float* __restrict__ mean_out,
                  float* __restrict__ rstd_out, int rows, int cols) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float c = *absmax_in * 0.125f;
    const float eps_eff = eps * c * c;
    const float inv_n = 1.0f / cols;
    float omax = 0.f;
    for (int row = blockIdx.x * WARPS + warp; row < rows; row += gridDim.x * WARPS) {
        const TIn* xr = x + (size_t)row * cols;
        float4 v[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int i = lane * 4 + j * 128;
            v[j] = i < cols ? ld4(xr + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < NV; ++j) s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
        const float mean = warp_sum(s) * inv_n;
        float ss = 0.f;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            if (lane * 4 + j * 128 < cols) {
                const float a = v[j].x - mean, b = v[j].y - mean, d = v[j].z - mean, e = v[j].w - mean;
                ss += (a * a + b * b) + (d * d + e * e);
            }
        }
        const float var = warp_sum(ss) * inv_n;
        const float rstd = rsqrtf(var + eps_eff);
        if (lane == 0 && mean_out != nullptr) {
            mean_out[row] = mean;
            rstd_out[row] = rstd;
        }
        TOut* orow = out + (size_t)row * cols;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int i = lane * 4 + j * 128;
            if (i < cols) {
                const float4 g = ld4(gamma + i), bt = ld4(beta + i);
                float4 y;
                y.x = (v[j].x - mean) * rstd * g.x + bt.x;
                y.y = (v[j].y - mean) * rstd * g.y + bt.y;
                y.z = (v[j].z - mean) * rstd * g.z + bt.z;
                y.w = (v[j].w - mean) * rstd * g.w + bt.w;
                if (RES) {
                    const float4 r = ld4(residual + (size_t)row * cols + i);
                    y.x += r.x; y.y += r.y; y.z += r.z; y.w += r.w;
                }
                st4(orow + i, y);
                if (absmax_out != nullptr) {
                    omax = fmaxf(omax, fmaxf(fmaxf(fabsf(round_as(y.x, orow)), fabsf(round_as(y.y, orow))),
                                             fmaxf(fabsf(round_as(y.z, orow)), fabsf(round_as(y.w, orow)))));
                }
            }
        }
    }
    if (absmax_out != nullptr) {
        omax = warp_max(omax);
        if (lane == 0 && omax > 0.f) atomic_max_nonneg(absmax_out, omax);
    }
}

// Backward.  dy: gradient of the LN output (TDy); dres (optional fp32): gradient already flowing on the
// residual path that must be added to dx (fp32 output) — used for the input/post-attention/final LNs.
//   dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)),  xhat = (x - mean) * rstd
// drop.p > 0: x was the output of a dropout site, so dx is masked as in ln_bwd_fused_kernel (same element counter).
template <typename TIn, typename TDy, typename TDx>
__global__ void __launch_bounds__(WARPS * 32)
ln_bwd_dx_kernel(const TIn* __restrict__ x, const TDy* __restrict__ dy, const float* __restrict__ mean_in,
                 const float* __restrict__ rstd_in, const __nv_bfloat16* __restrict__ gamma,
                 const float* __restrict__ dres, TDx* __restrict__ dx, int rows, int cols, const DropoutArgs drop) {
    extern __shared__ float smem_f[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* sx = smem_f + (size_t)warp * 2 * cols;   // xhat
    float* sg = sx + cols;                            // gamma * dy
    const float inv_n = 1.0f / cols;
    for (int row = blockIdx.x * WARPS + warp; row < rows; row += gridDim.x * WARPS) {
        const float mean = mean_in[row], rstd = rstd_in[row];
        const TIn* xr = x + (size_t)row * cols;
        const TDy* dyr = dy + (size_t)row * cols;
        float s1 = 0.f, s2 = 0.f;
        for (int i = lane * 4; i < cols; i += 128) {
            float4 v = ld4(xr + i), d = ld4(dyr + i), g = ld4(gamma + i);
            float4 xh = make_float4((v.x - mean) * rstd, (v.y - mean) * rstd, (v.z - mean) * rstd, (v.w - mean) * rstd);
            float4 a = make_float4(g.x * d.x, g.y * d.y, g.z * d.z, g.w * d.w);
            st4(sx + i, xh);
            st4(sg + i, a);
            s1 += (a.x + a.y) + (a.z + a.w);
            s2 += (a.x * xh.x + a.y * xh.y) + (a.z * xh.z + a.w * xh.w);
        }
        s1 = warp_sum(s1) * inv_n;
        s2 = warp_sum(s2) * inv_n;
        TDx* dxr = dx + (size_t)row * cols;
        for (int i = lane * 4; i < cols; i += 128) {
            float4 xh = ld4(sx + i), a = ld4(sg + i);
            float4 o;
            o.x = rstd * (a.x - s1 - xh.x * s2);
            o.y = rstd * (a.y - s1 - xh.y * s2);
            o.z = rstd * (a.z - s1 - xh.z * s2);
            o.w = rstd * (a.w - s1 - xh.w * s2);
            if (dres != nullptr) {
                float4 r = ld4(dres + (size_t)row * cols + i);
                o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
            }
            if (drop.p > 0.f) dropout4(drop, ((size_t)row * cols + i) >> 2, o.x, o.y, o.z, o.w);
            st4(dxr + i, o);
        }
        __syncwarp();
    }
}

// Fused backward (cols % 256 == 0): the CTA has cols/8 threads, each owning 8 fixed columns (two float4 groups), so
// its share of dgamma / dbeta lives in 16 registers for the whole kernel and the parameter gradients cost no extra
// pass.  Rows are processed 4 at a time: one block reduction (8 values) per 4 rows, every operand read exactly once.
constexpr int FB_R = 4;
template <typename TIn, typename TDy, typename TDx>
__global__ void __launch_bounds__(512)
ln_bwd_fused_kernel(const TIn* __restrict__ x, const TDy* __restrict__ dy, const float* __restrict__ mean_in,
                    const float* __restrict__ rstd_in, const __nv_bfloat16* __restrict__ gamma,
                    const float* __restrict__ dres, TDx* __restrict__ dx, float* __restrict__ partials, int rows,
                    int cols, int rows_per_cta, const DropoutArgs drop, int want_dxsum) {
    __shared__ float red[2][16][2 * FB_R];          // [buffer][warp][s1 x R, s2 x R]
    const int nwarps = blockDim.x >> 5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c0 = threadIdx.x * 4, c1 = c0 + cols / 2;
    const float4 g0 = ld4(gamma + c0), g1 = ld4(gamma + c1);
    float4 dg0 = make_float4(0.f, 0.f, 0.f, 0.f), dg1 = dg0, db0 = dg0, db1 = dg0;
    float4 ds0 = dg0, ds1 = dg0;                     // column sums of dx (= bias gradient of the GEMM that produced x)
    const float inv_n = 1.0f / cols;
    const int r_begin = blockIdx.x * rows_per_cta;
    const int r_end = min(rows, r_begin + rows_per_cta);
    int buf = 0;
    for (int r0 = r_begin; r0 < r_end; r0 += FB_R, buf ^= 1) {
        float4 xh0[FB_R], xh1[FB_R], a0[FB_R], a1[FB_R];
        float rs[FB_R];
        float part[2 * FB_R];
#pragma unroll
        for (int j = 0; j < FB_R; ++j) {
            const int row = r0 + j;
            const bool ok = row < r_end;
            const float mean = ok ? mean_in[row] : 0.f;
            rs[j] = ok ? rstd_in[row] : 0.f;
            const size_t off = (size_t)(ok ? row : r_begin) * cols;
            const float4 v0 = ld4(x + off + c0), v1 = ld4(x + off + c1);
            float4 d0 = ld4(dy + off + c0), d1 = ld4(dy + off + c1);
            if (!ok) { d0 = make_float4(0.f, 0.f, 0.f, 0.f); d1 = d0; }
            xh0[j] = make_float4((v0.x - mean) * rs[j], (v0.y - mean) * rs[j], (v0.z - mean) * rs[j], (v0.w - mean) * rs[j]);
            xh1[j] = make_float4((v1.x - mean) * rs[j], (v1.y - mean) * rs[j], (v1.z - mean) * rs[j], (v1.w - mean) * rs[j]);
            a0[j] = make_float4(g0.x * d0.x, g0.y * d0.y, g0.z * d0.z, g0.w * d0.w);
            a1[j] = make_float4(g1.x * d1.x, g1.y * d1.y, g1.z * d1.z, g1.w * d1.w);
            dg0.x += d0.x * xh0[j].x; dg0.y += d0.y * xh0[j].y; dg0.z += d0.z * xh0[j].z; dg0.w += d0.w * xh0[j].w;
            dg1.x += d1.x * xh1[j].x; dg1.y += d1.y * xh1[j].y; dg1.z += d1.z * xh1[j].z; dg1.w += d1.w * xh1[j].w;
            db0.x += d0.x; db0.y += d0.y; db0.z += d0.z; db0.w += d0.w;
            db1.x += d1.x; db1.y += d1.y; db1.z += d1.z; db1.w += d1.w;
            part[j] = (a0[j].x + a0[j].y) + (a0[j].z + a0[j].w) + (a1[j].x + a1[j].y) + (a1[j].z + a1[j].w);
            part[FB_R + j] = (a0[j].x * xh0[j].x + a0[j].y * xh0[j].y) + (a0[j].z * xh0[j].z + a0[j].w * xh0[j].w) +
                             (a1[j].x * xh1[j].x + a1[j].y * xh1[j].y) + (a1[j].z * xh1[j].z + a1[j].w * xh1[j].w);
        }
#pragma unroll
        for (int t = 0; t < 2 * FB_R; ++t) part[t] = warp_sum(part[t]);
        if (lane == 0) {
#pragma unroll
            for (int t = 0; t < 2 * FB_R; ++t) red[buf][warp][t] = part[t];
        }
        __syncthreads();
#pragma unroll
        for (int t = 0; t < 2 * FB_R; ++t) {
            float acc = 0.f;
            for (int w = 0; w < nwarps; ++w) acc += red[buf][w][t];
            part[t] = acc * inv_n;
        }
#pragma unroll
        for (int j = 0; j < FB_R; ++j) {
            const int row = r0 + j;
            if (row < r_end) {
                const float s1 = part[j], s2 = part[FB_R + j];
                const size_t off = (size_t)row * cols;
                float4 o0, o1;
                o0.x = rs[j] * (a0[j].x - s1 - xh0[j].x * s2); o0.y = rs[j] * (a0[j].y - s1 - xh0[j].y * s2);
                o0.z = rs[j] * (a0[j].z - s1 - xh0[j].z * s2); o0.w = rs[j] * (a0[j].w - s1 - xh0[j].w * s2);
                o1.x = rs[j] * (a1[j].x - s1 - xh1[j].x * s2); o1.y = rs[j] * (a1[j].y - s1 - xh1[j].y * s2);
                o1.z = rs[j] * (a1[j].z - s1 - xh1[j].z * s2); o1.w = rs[j] * (a1[j].w - s1 - xh1[j].w * s2);
                if (dres != nullptr) {
                    const float4 q0 = ld4(dres + off + c0), q1 = ld4(dres + off + c1);
                    o0.x += q0.x; o0.y += q0.y; o0.z += q0.z; o0.w += q0.w;
                    o1.x += q1.x; o1.y += q1.y; o1.z += q1.z; o1.w += q1.w;
                }
                if (drop.p > 0.f) {   // x was the output of a dropout site: dx flows back through the same mask
                    dropout4(drop, (off + c0) >> 2, o0.x, o0.y, o0.z, o0.w);
                    dropout4(drop, (off + c1) >> 2, o1.x, o1.y, o1.z, o1.w);
                }
                st4(dx + off + c0, o0);
                st4(dx + off + c1, o1);
                if (want_dxsum) {   // summed as stored (rounded to the output type), like a separate column-sum pass
                    ds0.x += round_as(o0.x, dx); ds0.y += round_as(o0.y, dx); ds0.z += round_as(o0.z, dx); ds0.w += round_as(o0.w, dx);
                    ds1.x += round_as(o1.x, dx); ds1.y += round_as(o1.y, dx); ds1.z += round_as(o1.z, dx); ds1.w += round_as(o1.w, dx);
                }
            }
        }
    }
    const int nacc = want_dxsum ? 3 : 2;
    float* pout = partials + (size_t)blockIdx.x * nacc * cols;
    st4(pout + c0, dg0); st4(pout + c1, dg1);
    st4(pout + cols + c0, db0); st4(pout + cols + c1, db1);
    if (want_dxsum) { st4(pout + 2 * cols + c0, ds0); st4(pout + 2 * cols + c1, ds1); }
}

// reduces [nparts][nacc][cols] partials into up to three bf16 vectors; block = 32 columns x 8 part groups
__global__ void __launch_bounds__(256)
ln_bwd_finalize3_kernel(const float* __restrict__ partials, int nparts, int cols, int nacc,
                        __nv_bfloat16* __restrict__ o0, __nv_bfloat16* __restrict__ o1,
                        __nv_bfloat16* __restrict__ o2) {
    __shared__ float sh[8][32];
    const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + lane;                    // index into [nacc][cols]
    float s0 = 0.f, s1 = 0.f;
    if (i < nacc * cols) {
        const size_t stride = (size_t)nacc * cols;
        int p = grp;
        for (; p + 8 < nparts; p += 16) {
            s0 += partials[(size_t)p * stride + i];
            s1 += partials[(size_t)(p + 8) * stride + i];
        }
        if (p < nparts) s0 += partials[(size_t)p * stride + i];
    }
    sh[grp][lane] = s0 + s1;
    __syncthreads();
    if (grp == 0 && i < nacc * cols) {
        float s = 0.f;
#pragma unroll
        for (int g = 0; g < 8; ++g) s += sh[g][lane];
        const int which = i / cols, c = i - which * cols;
        (which == 0 ? o0 : (which == 1 ? o1 : o2))[c] = __float2bfloat16_rn(s);
    }
}

// dgamma[c] = sum_r dy[r,c] * xhat[r,c], dbeta[c] = sum_r dy[r,c].  Thread per column (coalesced across columns),
// rows split over blockIdx.y; partial sums go to `partials` [gridDim.y, 2, cols], reduced by ln_bwd_finalize.
constexpr int PARAM_ROW_SPLITS = 32;
template <typename TIn, typename TDy>
__global__ void __launch_bounds__(128)
ln_bwd_param_kernel(const TIn* __restrict__ x, const TDy* __restrict__ dy, const float* __restrict__ mean_in,
                    const float* __restrict__ rstd_in, float* __restrict__ partials, int rows, int cols) {
    const int c = blockIdx.x * 128 + threadIdx.x;
    const int rows_per = (rows + gridDim.y - 1) / gridDim.y;
    const int r0 = blockIdx.y * rows_per;
    const int r1 = min(rows, r0 + rows_per);
    float dg = 0.f, db = 0.f;
    if (c < cols) {
#pragma unroll 4
        for (int r = r0; r < r1; ++r) {
            const float d = ld_as_float(dy, (size_t)r * cols + c);
            const float xh = (ld_as_float(x, (size_t)r * cols + c) - mean_in[r]) * rstd_in[r];
            dg += d * xh;
            db += d;
        }
        partials[((size_t)blockIdx.y * 2 + 0) * cols + c] = dg;
        partials[((size_t)blockIdx.y * 2 + 1) * cols + c] = db;
    }
}

__global__ void ln_bwd_finalize_kernel(const float* __restrict__ partials, int nparts, int cols,
                                       __nv_bfloat16* __restrict__ dgamma, __nv_bfloat16* __restrict__ dbeta) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * cols) return;
    float s = 0.f;
    for (int p = 0; p < nparts; ++p) s += partials[(size_t)p * 2 * cols + i];
    if (i < cols) dgamma[i] = __float2bfloat16_rn(s);
    else dbeta[i - cols] = __float2bfloat16_rn(s);
}

int fwd_grid(int rows) {
    int blocks = (rows + WARPS - 1) / WARPS;
    int cap = cvh::num_sms() * 4;
    return blocks < cap ? blocks : cap;
}

}  // namespace

extern "C" int cv_layernorm_absmax_fwd(const void* x, int x_is_bf16, const float* absmax_in, const void* gamma,
                                       const void* beta, float eps, const float* residual, void* out,
                                       int out_is_bf16, float* absmax_out, float* mean_out, float* rstd_out,
                                       int rows, int cols, void* stream) {
    CV_REQUIRE(x && absmax_in && gamma && beta && out, "null pointer");
    CV_REQUIRE(rows > 0 && cols > 0 && cols % 4 == 0, "cols must be a positive multiple of 4");
    CV_REQUIRE((mean_out == nullptr) == (rstd_out == nullptr), "mean_out and rstd_out go together");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t smem = (size_t)WARPS * cols * sizeof(float);
    CV_REQUIRE(smem <= 200 * 1024, "hidden size too large for the row cache");
    const int grid = fwd_grid(rows);
    const __nv_bfloat16* g = static_cast<const __nv_bfloat16*>(gamma);
    const __nv_bfloat16* b = static_cast<const __nv_bfloat16*>(beta);
    static int reg_rows = -1;                            // COGVIEW_B200_LN_REG=0: the shared-memory staged kernel only
    if (reg_rows < 0) {
        const char* e = getenv("COGVIEW_B200_LN_REG");
        reg_rows = (e && e[0] == '0') ? 0 : 1;
    }
    // the register kernel serves rows without a residual; with one, the staged kernel is used (tools/ln_time.py times both)
    const bool use_reg = reg_rows && cols <= 128 * 20 && residual == nullptr;
    int rgrid = 2 * cvh::num_sms();                      // two CTAs of 8 warps per SM, rows grid-strided
    if (rgrid > (rows + WARPS - 1) / WARPS) rgrid = (rows + WARPS - 1) / WARPS;
#define LAUNCH(TI, TO, RES)                                                                                    \
    do {                                                                                                       \
        if (use_reg) {                                                                                         \
            ln_fwd_reg_kernel<TI, TO, RES, 20><<<rgrid, WARPS * 32, 0, s>>>(                                   \
                static_cast<const TI*>(x), absmax_in, g, b, eps, residual, static_cast<TO*>(out), absmax_out,  \
                mean_out, rstd_out, rows, cols);                                                               \
            break;                                                                                             \
        }                                                                                                      \
        auto k = ln_fwd_kernel<TI, TO, RES>;                                                                   \
        CV_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));              \
        k<<<grid, WARPS * 32, smem, s>>>(static_cast<const TI*>(x), absmax_in, g, b, eps, residual,            \
                                         static_cast<TO*>(out), absmax_out, mean_out, rstd_out, rows, cols);   \
    } while (0)
    const bool res = residual != nullptr;
    if (!x_is_bf16 && out_is_bf16 && !res) LAUNCH(float, __nv_bfloat16, false);
    else if (x_is_bf16 && !out_is_bf16 && res) LAUNCH(__nv_bfloat16, float, true);
    else if (x_is_bf16 && out_is_bf16 && !res) LAUNCH(__nv_bfloat16, __nv_bfloat16, false);
    else if (!x_is_bf16 && !out_is_bf16 && !res) LAUNCH(float, float, false);
    else if (!x_is_bf16 && !out_is_bf16 && res) LAUNCH(float, float, true);
    else return cvh::fail_arg(__func__, "unsupported dtype/residual combination");
#undef LAUNCH
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int64_t cv_layernorm_bwd_workspace_bytes(int rows, int cols) {
    (void)rows;
    const int64_t parts = 2 * cvh::num_sms() > PARAM_ROW_SPLITS ? 2 * cvh::num_sms() : PARAM_ROW_SPLITS;
    return parts * 3 * cols * sizeof(float);
}

extern "C" int cv_layernorm_absmax_bwd(const void* x, int x_is_bf16, const void* dy, int dy_is_bf16,
                                       const float* mean, const float* rstd, const void* gamma, const float* dres,
                                       void* dx, int dx_is_bf16, void* dgamma, void* dbeta, float* workspace,
                                       int rows, int cols, float dropout_p, uint64_t seed, uint32_t site,
                                       void* dxsum, void* stream) {
    const cvh::HostDropout hd = cvh::make_dropout(dropout_p, seed, site);
    DropoutArgs dargs;
    dargs.p = hd.p; dargs.scale = hd.scale; dargs.threshold = hd.threshold; dargs.stream = hd.stream; dargs.seed = hd.seed;
    CV_REQUIRE(x && dy && mean && rstd && gamma && dx && dgamma && dbeta && workspace, "null pointer");
    CV_REQUIRE(rows > 0 && cols > 0 && cols % 4 == 0, "cols must be a positive multiple of 4");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const __nv_bfloat16* g = static_cast<const __nv_bfloat16*>(gamma);
    // fused path (parameter gradients in registers, every operand read once)
    if (cols % 256 == 0 && cols / 8 <= 512) {
        const int threads = cols / 8;
        int fgrid = cvh::num_sms();          // 128 registers x cols/8 threads: one CTA per SM
        int rows_per_cta = (rows + fgrid - 1) / fgrid;
        rows_per_cta = (rows_per_cta + FB_R - 1) / FB_R * FB_R;
        fgrid = (rows + rows_per_cta - 1) / rows_per_cta;
#define LAUNCH_F(TI, TDY, TDX)                                                                                 \
    ln_bwd_fused_kernel<TI, TDY, TDX><<<fgrid, threads, 0, s>>>(static_cast<const TI*>(x), static_cast<const TDY*>(dy), \
                                                                mean, rstd, g, dres, static_cast<TDX*>(dx), workspace,   \
                                                                rows, cols, rows_per_cta, dargs, dxsum != nullptr)
        if (x_is_bf16 && !dy_is_bf16 && dx_is_bf16) LAUNCH_F(__nv_bfloat16, float, __nv_bfloat16);
        else if (!x_is_bf16 && dy_is_bf16 && !dx_is_bf16) LAUNCH_F(float, __nv_bfloat16, float);
        else if (!x_is_bf16 && !dy_is_bf16 && !dx_is_bf16) LAUNCH_F(float, float, float);
        else if (x_is_bf16 && dy_is_bf16 && dx_is_bf16) LAUNCH_F(__nv_bfloat16, __nv_bfloat16, __nv_bfloat16);
        else return cvh::fail_arg(__func__, "unsupported dtype combination");
#undef LAUNCH_F
        CV_LAUNCH_CHECK();
        const int nacc = dxsum != nullptr ? 3 : 2;
        ln_bwd_finalize3_kernel<<<(nacc * cols + 31) / 32, 256, 0, s>>>(workspace, fgrid, cols, nacc,
                                                                         static_cast<__nv_bfloat16*>(dgamma),
                                                                         static_cast<__nv_bfloat16*>(dbeta),
                                                                         static_cast<__nv_bfloat16*>(dxsum));
        CV_LAUNCH_CHECK();
        return 0;
    }
    CV_REQUIRE(dxsum == nullptr, "the column sum of dx is only produced by the fused path (hidden size % 256 == 0)");
    // the unfused dx kernel stages two fp32 rows per warp in shared memory
    const size_t smem = (size_t)WARPS * 2 * cols * sizeof(float);
    CV_REQUIRE(smem <= 220 * 1024, "hidden size too large for the row cache");
    const int grid = fwd_grid(rows);
    const int splits = rows < PARAM_ROW_SPLITS ? rows : PARAM_ROW_SPLITS;
    dim3 pgrid((cols + 127) / 128, splits);
#define LAUNCH(TI, TDY, TDX)                                                                                   \
    do {                                                                                                       \
        auto k = ln_bwd_dx_kernel<TI, TDY, TDX>;                                                               \
        CV_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));              \
        k<<<grid, WARPS * 32, smem, s>>>(static_cast<const TI*>(x), static_cast<const TDY*>(dy), mean, rstd, g, \
                                         dres, static_cast<TDX*>(dx), rows, cols, dargs);                      \
        ln_bwd_param_kernel<TI, TDY><<<pgrid, 128, 0, s>>>(static_cast<const TI*>(x), static_cast<const TDY*>(dy), \
                                                           mean, rstd, workspace, rows, cols);                  \
    } while (0)
    if (x_is_bf16 && !dy_is_bf16 && dx_is_bf16) LAUNCH(__nv_bfloat16, float, __nv_bfloat16);       // third/fourth LN
    else if (!x_is_bf16 && dy_is_bf16 && !dx_is_bf16) LAUNCH(float, __nv_bfloat16, float);         // input/post/final LN
    else if (!x_is_bf16 && !dy_is_bf16 && !dx_is_bf16) LAUNCH(float, float, float);
    else if (x_is_bf16 && dy_is_bf16 && dx_is_bf16) LAUNCH(__nv_bfloat16, __nv_bfloat16, __nv_bfloat16);
    else return cvh::fail_arg(__func__, "unsupported dtype combination");
#undef LAUNCH
    CV_LAUNCH_CHECK();
    const int n = 2 * cols;
    ln_bwd_finalize_kernel<<<(n + 255) / 256, 256, 0, s>>>(workspace, splits, cols, static_cast<__nv_bfloat16*>(dgamma),
                                                          static_cast<__nv_bfloat16*>(dbeta));
    CV_LAUNCH_CHECK();
    return 0;
}
