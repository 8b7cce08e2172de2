// VQ-VAE quantiser and the HBM-bound ends of the image tokenizer.
//
//   cv_vq_split3      z (fp32) -> [hi | hi | lo] bf16 so that ONE bf16 tensor-core GEMM against the codebook packed as
//                     [hi | lo | hi] accumulates z_hi.E_hi + z_hi.E_lo + z_lo.E_hi in fp32 (16 mantissa bits per operand)
//   cv_vq_argmin      argmin_j ||E_j||^2 - 2 z.E_j over the score matrix (the row-constant ||z||^2 of
//                     Quantize.forward_, /root/reference/vqvae/vqvae_zc.py:43-51, is dropped), first index on ties,
//                     with exact fp32 re-scoring of the two best codes when their gap is inside the split's error
//   cv_vq_lookup      embed_code (vqvae_zc.py:95-96) fused with the NHWC layout the decoder reads
//   cv_im2col_k4s2_c3 patches of the 3-channel image for the first encoder conv (vqvae_zc.py:122; Cin=3 is HBM-bound,
//                     so it runs as im2col(K=48 padded to 64) + cv_gemm_bf16 with a ReLU epilogue)
//   cv_conv1x1_out3   the decoder's last 1x1 conv 512->3 (vqvae_zc.py:191) fused with the de-normalisation of
//                     vqvae/api.py:43 and the NHWC->NCHW fp32 output
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

__global__ void vq_split3_kernel(const float* __restrict__ z, __nv_bfloat16* __restrict__ out, size_t rows, int dim) {
    const size_t n = rows * (size_t)dim;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / dim;
        const int c = (int)(i - r * dim);
        const float v = z[i];
        const __nv_bfloat16 hi = __float2bfloat16_rn(v);
        const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
        __nv_bfloat16* o = out + r * 3 * dim;
        o[c] = hi;
        o[dim + c] = hi;
        o[2 * dim + c] = lo;
    }
}

constexpr int AM_THREADS = 256;
struct Best { float v0; int i0; float v1; int i1; };   // best and second-best (value, index)

__device__ __forceinline__ void best_insert(Best& b, float v, int i) {
    if (v < b.v0 || (v == b.v0 && i < b.i0)) { b.v1 = b.v0; b.i1 = b.i0; b.v0 = v; b.i0 = i; }
    else if (v < b.v1 || (v == b.v1 && i < b.i1)) { b.v1 = v; b.i1 = i; }
}
__device__ __forceinline__ Best best_merge(Best a, const Best& o) {
    best_insert(a, o.v0, o.i0);
    best_insert(a, o.v1, o.i1);
    return a;
}

__global__ void __launch_bounds__(AM_THREADS)
vq_argmin_kernel(const float* __restrict__ scores, int64_t ld, const float* __restrict__ e2,
                 const float* __restrict__ z, const float* __restrict__ codebook /*[n_embed, dim]*/,
                 int64_t* __restrict__ idx_out, int n_embed, int dim, float margin) {
    __shared__ Best sh[AM_THREADS / 32];
    __shared__ float sdot[2];
    const int row = blockIdx.x;
    const float* s = scores + (size_t)row * ld;
    Best b = {INFINITY, 0x7fffffff, INFINITY, 0x7fffffff};
    for (int j = threadIdx.x * 4; j < n_embed; j += AM_THREADS * 4) {
        const float4 sv = *reinterpret_cast<const float4*>(s + j);
        const float4 ev = *reinterpret_cast<const float4*>(e2 + j);
        best_insert(b, ev.x - 2.f * sv.x, j);
        best_insert(b, ev.y - 2.f * sv.y, j + 1);
        best_insert(b, ev.z - 2.f * sv.z, j + 2);
        best_insert(b, ev.w - 2.f * sv.w, j + 3);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Best t;
        t.v0 = __shfl_xor_sync(0xffffffffu, b.v0, o); t.i0 = __shfl_xor_sync(0xffffffffu, b.i0, o);
        t.v1 = __shfl_xor_sync(0xffffffffu, b.v1, o); t.i1 = __shfl_xor_sync(0xffffffffu, b.i1, o);
        b = best_merge(b, t);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) sh[warp] = b;
    __syncthreads();
    if (warp == 0) {
        Best t = lane < AM_THREADS / 32 ? sh[lane] : Best{INFINITY, 0x7fffffff, INFINITY, 0x7fffffff};
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            Best u;
            u.v0 = __shfl_xor_sync(0xffffffffu, t.v0, o); u.i0 = __shfl_xor_sync(0xffffffffu, t.i0, o);
            u.v1 = __shfl_xor_sync(0xffffffffu, t.v1, o); u.i1 = __shfl_xor_sync(0xffffffffu, t.i1, o);
            t = best_merge(t, u);
        }
        if (lane == 0) sh[0] = t;
    }
    __syncthreads();
    b = sh[0];
    int winner = b.i0;
    const bool close = (b.v1 - b.v0) < margin * fmaxf(1.f, fabsf(b.v0));
    if (close && b.i1 < n_embed) {
        // exact fp32 distances of the two candidates: ||E_j||^2 - 2 z.E_j with fp32 FMAs (warps 0 and 1)
        if (warp < 2) {
            const int j = warp == 0 ? b.i0 : b.i1;
            const float* zr = z + (size_t)row * dim;
            const float* er = codebook + (size_t)j * dim;
            float acc = 0.f;
            for (int k = lane; k < dim; k += 32) acc = fmaf(er[k], er[k] - 2.f * zr[k], acc);
            acc = warp_sum(acc);
            if (lane == 0) sdot[warp] = acc;
        }
        __syncthreads();
        const float d0 = sdot[0], d1 = sdot[1];
        if (d1 < d0 || (d1 == d0 && b.i1 < b.i0)) winner = b.i1;
    }
    if (threadIdx.x == 0) idx_out[row] = winner;
}

__global__ void vq_lookup_kernel(const int64_t* __restrict__ idx, const float* __restrict__ codebook,
                                 __nv_bfloat16* __restrict__ out_bf16, float* __restrict__ out_f32, size_t rows,
                                 int dim) {
    const size_t n = rows * (size_t)(dim / 4);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / (dim / 4);
        const int c = (int)(i - r * (dim / 4)) * 4;
        const float4 v = *reinterpret_cast<const float4*>(codebook + (size_t)idx[r] * dim + c);
        if (out_bf16 != nullptr) {
            uint2 u;
            u.x = pack_bf16x2(v.x, v.y);
            u.y = pack_bf16x2(v.z, v.w);
            *reinterpret_cast<uint2*>(out_bf16 + r * dim + c) = u;
        }
        if (out_f32 != nullptr) *reinterpret_cast<float4*>(out_f32 + r * dim + c) = v;
    }
}

// out[(b, oy, ox), (ky*4+kx)*3 + c] = img[b, c, 2oy-1+ky, 2ox-1+kx] (zero outside), columns 48..63 zero
__global__ void im2col_k4s2_c3_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out, int B, int H,
                                      int W) {
    const int OH = H / 2, OW = W / 2;
    const size_t npix = (size_t)B * OH * OW;
    for (size_t pix = blockIdx.x * (size_t)blockDim.x + threadIdx.x; pix < npix;
         pix += (size_t)gridDim.x * blockDim.x) {
        const int ox = (int)(pix % OW);
        const int oy = (int)((pix / OW) % OH);
        const int b = (int)(pix / ((size_t)OW * OH));
        uint32_t packed[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) packed[i] = 0;
        const float* base = img + (size_t)b * 3 * H * W;
#pragma unroll
        for (int ky = 0; ky < 4; ++ky) {
            const int iy = 2 * oy - 1 + ky;
#pragma unroll
            for (int kx = 0; kx < 4; ++kx) {
                const int ix = 2 * ox - 1 + kx;
                const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const int k = (ky * 4 + kx) * 3 + c;
                    const float v = in ? base[((size_t)c * H + iy) * W + ix] : 0.f;
                    const uint32_t bits = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v));
                    packed[k >> 1] |= (k & 1) ? (bits << 16) : bits;
                }
            }
        }
        uint4* o = reinterpret_cast<uint4*>(out + pix * 64);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
    }
}

// out[b, c, y, x] = (sum_k x[(b,y,x), k] * w[c, k] + bias[c]) * scale[c] + shift[c]   (the decoder's last 1x1 convolution,
// vqvae/vqvae_zc.py:181-192, + the de-normalisation of api.code2img).  HBM bound: 2 cin bytes in, 12 bytes out per pixel.
// 8 lanes per pixel, 4 pixels per warp: lane `sub` owns channels 8 sub + 64 j + t (t < 8), so the 8 lanes of a pixel read
// 128 contiguous bytes per step and up to 8 steps (1 KB per pixel at cin = 512) are in flight per lane; the 3 x cin weights
// sit in shared memory.  (The first version gave a whole warp to ONE pixel at a time — 15 shuffles and 2 loads per pixel —
// and kept too few loads in flight to approach the HBM bandwidth.)
constexpr int C1_MAXJ = 8;      // cin <= 512 in one pass; larger cin loops
__global__ void __launch_bounds__(256)
conv1x1_out3_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                    const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ out,
                    size_t npix, int hw, int cin) {
    extern __shared__ float w_s[];                 // [3][cin]
    for (int i = threadIdx.x; i < 3 * cin; i += blockDim.x) w_s[i] = w[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, sub = lane & 7, pl = lane >> 3;
    const size_t warp_global = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    const int nj = cin / 64;                       // 16-byte steps per lane (cin % 64 == 0)
    const float b0 = bias[0], b1 = bias[1], b2 = bias[2];
    const float s0 = scale[0], s1 = scale[1], s2 = scale[2], t0 = shift[0], t1 = shift[1], t2 = shift[2];
    for (size_t p0 = warp_global * 4; p0 < npix; p0 += nwarps * 4) {
        const size_t pix = p0 + pl;
        const bool ok = pix < npix;
        const __nv_bfloat16* xr = x + (ok ? pix : p0) * cin + sub * 8;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int j0 = 0; j0 < nj; j0 += C1_MAXJ) {
            uint4 u[C1_MAXJ];
#pragma unroll
            for (int j = 0; j < C1_MAXJ; ++j)
                u[j] = (j0 + j < nj) ? *reinterpret_cast<const uint4*>(xr + (j0 + j) * 64) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int j = 0; j < C1_MAXJ; ++j) {
                if (j0 + j < nj) {
                    const int k = (j0 + j) * 64 + sub * 8;
                    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u[j]);
                    float v[8];
#pragma unroll
                    for (int t = 0; t < 4; ++t) { v[2 * t] = __low2float(h2[t]); v[2 * t + 1] = __high2float(h2[t]); }
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float4 wa = *reinterpret_cast<const float4*>(w_s + c * cin + k);
                        const float4 wb = *reinterpret_cast<const float4*>(w_s + c * cin + k + 4);
                        float acc = c == 0 ? a0 : (c == 1 ? a1 : a2);
                        acc = fmaf(v[0], wa.x, acc); acc = fmaf(v[1], wa.y, acc); acc = fmaf(v[2], wa.z, acc);
                        acc = fmaf(v[3], wa.w, acc); acc = fmaf(v[4], wb.x, acc); acc = fmaf(v[5], wb.y, acc);
                        acc = fmaf(v[6], wb.z, acc); acc = fmaf(v[7], wb.w, acc);
                        if (c == 0) a0 = acc; else if (c == 1) a1 = acc; else a2 = acc;
                    }
                }
            }
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {          // sum over the 8 lanes of the pixel
            a0 += __shfl_xor_sync(0xffffffffu, a0, o);
            a1 += __shfl_xor_sync(0xffffffffu, a1, o);
            a2 += __shfl_xor_sync(0xffffffffu, a2, o);
        }
        if (ok && sub == 0) {
            const size_t b = pix / hw, rem = pix % hw;
            float* o = out + b * 3 * hw + rem;
            o[0] = (a0 + b0) * s0 + t0;
            o[hw] = (a1 + b1) * s1 + t1;
            o[2 * (size_t)hw] = (a2 + b2) * s2 + t2;
        }
    }
}

int grid_for(size_t items, int threads) {
    size_t blocks = (items + threads - 1) / threads;
    size_t cap = (size_t)cvh::num_sms() * 16;
    return (int)(blocks < cap ? (blocks ? blocks : 1) : cap);
}
}  // namespace

extern "C" int cv_vq_split3(const float* z, void* out, int64_t rows, int dim, void* stream) {
    CV_REQUIRE(z && out && rows > 0 && dim > 0, "bad argument");
    vq_split3_kernel<<<grid_for((size_t)rows * dim, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        z, static_cast<__nv_bfloat16*>(out), (size_t)rows, dim);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_vq_argmin(const float* scores, int64_t ld, const float* e2, const float* z, const float* codebook,
                            int64_t* idx_out, int64_t rows, int n_embed, int dim, float margin, void* stream) {
    CV_REQUIRE(scores && e2 && z && codebook && idx_out, "null pointer");
    CV_REQUIRE(rows > 0 && n_embed % 4 == 0 && ld % 4 == 0, "n_embed and ld must be multiples of 4");
    vq_argmin_kernel<<<(unsigned)rows, AM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        scores, ld, e2, z, codebook, idx_out, n_embed, dim, margin);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_vq_lookup(const int64_t* idx, const float* codebook, void* out_bf16, float* out_f32, int64_t rows,
                            int dim, void* stream) {
    CV_REQUIRE(idx && codebook && (out_bf16 || out_f32) && rows > 0 && dim % 4 == 0, "bad argument");
    vq_lookup_kernel<<<grid_for((size_t)rows * dim / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        idx, codebook, static_cast<__nv_bfloat16*>(out_bf16), out_f32, (size_t)rows, dim);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_im2col_k4s2_c3(const float* img, void* out, int B, int H, int W, void* stream) {
    CV_REQUIRE(img && out && B > 0 && H % 2 == 0 && W % 2 == 0, "bad argument");
    const size_t npix = (size_t)B * (H / 2) * (W / 2);
    im2col_k4s2_c3_kernel<<<grid_for(npix, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        img, static_cast<__nv_bfloat16*>(out), B, H, W);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_conv1x1_out3(const void* x, const float* w, const float* bias, const float* scale, const float* shift,
                               float* out, int B, int H, int W, int cin, void* stream) {
    CV_REQUIRE(x && w && bias && scale && shift && out, "null pointer");
    CV_REQUIRE(cin % 64 == 0 && cin <= 4096 && B > 0 && H > 0 && W > 0, "cin must be a multiple of 64 (<= 4096)");
    const size_t npix = (size_t)B * H * W;
    conv1x1_out3_kernel<<<grid_for((npix + 3) / 4 * 32, 256), 256, (size_t)3 * cin * sizeof(float),
                          static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), w, bias, scale, shift, out, npix, H * W, cin);
    CV_LAUNCH_CHECK();
    return 0;
}
