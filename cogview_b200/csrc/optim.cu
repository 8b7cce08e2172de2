// cv_adamw_step_multi: fused AdamW on bf16 parameters with fp32 master weights and moments.
//
// Replaces the optimizer sweep of the reference's training step: FP16_Optimizer.step (fp16/fp16.py:399-453:
// copy fp16 grads to fp32 masters' .grad, unscale, step, copy masters back to fp16) around apex FusedAdam
// (pretrain_gpt2.py:139-140; apex default adam_w_mode=True -> decoupled weight decay).  One pass:
//   g = grad * grad_scale (grad_scale carries the clip coefficient; bf16 needs no loss scale)
//   m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2
//   w = w - lr * ( (m / (1-b1^t)) / (sqrt(v / (1-b2^t)) + eps) + wd * w );   param_bf16 = round(w)
// HBM-bound: 2+2+12 bytes read, 2+12 written per parameter; 16-byte vectorised.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

// clip coefficient from the accumulated sum of squares: coef = min(1, max_norm / (sqrt(sumsq) + 1e-6)).
// A non-finite norm (one inf / NaN gradient anywhere) marks the step as skipped — the overflow branch of the
// reference's FP16_Optimizer.step (fp16/fp16.py:399-420): state[0] = 1 and the applied-step counter state[1] is not
// advanced; adamw_multi_kernel then leaves parameters, masters and moments untouched.
__global__ void clip_coef_kernel(const float* __restrict__ sumsq, float max_norm, float* __restrict__ coef,
                                 float* __restrict__ norm_out, int* __restrict__ state) {
    const float nrm = sqrtf(*sumsq);
    if (norm_out) *norm_out = nrm;
    const bool bad = !isfinite(nrm);
    const float c = max_norm / (nrm + 1e-6f);
    *coef = bad ? 0.f : ((max_norm > 0.f && c < 1.f) ? c : 1.f);
    if (state) {
        state[0] = bad ? 1 : 0;
        if (!bad) state[1] += 1;
    }
}

// ---- multi-tensor variants: one launch for the whole parameter list (a 4B model has ~780 tensors, most of them
// 2560-element vectors whose individual launches are latency-bound).  blockIdx.y = tensor, blockIdx.x strides.
constexpr int MT_CTAS = 32;

__global__ void __launch_bounds__(256)
adamw_multi_kernel(const cv_adamw_entry* __restrict__ table, float beta1, float beta2, float eps,
                   const float* __restrict__ grad_scale_dev, float grad_scale, const int* __restrict__ state) {
    if (state != nullptr && state[0] != 0) return;        // skipped step (non-finite gradient norm)
    const cv_adamw_entry e = table[blockIdx.y];
    const size_t n = (size_t)e.n, n4 = n / 4;
    if ((size_t)blockIdx.x * 256 >= n4 + 1) return;
    const float gs = grad_scale_dev ? *grad_scale_dev * grad_scale : grad_scale;
    __nv_bfloat16* param = static_cast<__nv_bfloat16*>(e.param);
    const __nv_bfloat16* grad = static_cast<const __nv_bfloat16*>(e.grad);
    float *master = e.master, *m = e.m, *v = e.v;
    const float lr = e.lr, weight_decay = e.weight_decay;
    float bc1 = e.bias_correction1, bc2 = e.bias_correction2;
    if (state != nullptr) {                                // bias correction from the count of APPLIED steps
        const float st = (float)state[1];
        bc1 = 1.f - powf(beta1, st);
        bc2 = 1.f - powf(beta2, st);
    }
    for (size_t i = blockIdx.x * (size_t)256 + threadIdx.x; i < n4; i += (size_t)gridDim.x * 256) {
        uint2 gu = reinterpret_cast<const uint2*>(grad)[i];
        const __nv_bfloat162* gp = reinterpret_cast<const __nv_bfloat162*>(&gu);
        float g[4] = {__low2float(gp[0]) * gs, __high2float(gp[0]) * gs, __low2float(gp[1]) * gs,
                      __high2float(gp[1]) * gs};
        float4 w4 = reinterpret_cast<float4*>(master)[i];
        float4 m4 = reinterpret_cast<float4*>(m)[i];
        float4 v4 = reinterpret_cast<float4*>(v)[i];
        float w[4] = {w4.x, w4.y, w4.z, w4.w}, mm[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            mm[t] = beta1 * mm[t] + (1.f - beta1) * g[t];
            vv[t] = beta2 * vv[t] + (1.f - beta2) * g[t] * g[t];
            const float upd = (mm[t] / bc1) / (sqrtf(vv[t] / bc2) + eps) + weight_decay * w[t];
            w[t] -= lr * upd;
        }
        reinterpret_cast<float4*>(master)[i] = make_float4(w[0], w[1], w[2], w[3]);
        reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
        reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
        uint2 pu;
        pu.x = pack_bf16x2(w[0], w[1]);
        pu.y = pack_bf16x2(w[2], w[3]);
        reinterpret_cast<uint2*>(param)[i] = pu;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const size_t i = n4 * 4 + threadIdx.x;
        const float g = __bfloat162float(grad[i]) * gs;
        float mm = beta1 * m[i] + (1.f - beta1) * g;
        float vv = beta2 * v[i] + (1.f - beta2) * g * g;
        float w = master[i];
        w -= lr * ((mm / bc1) / (sqrtf(vv / bc2) + eps) + weight_decay * w);
        m[i] = mm; v[i] = vv; master[i] = w;
        param[i] = __float2bfloat16_rn(w);
    }
}

__global__ void __launch_bounds__(256)
sumsq_multi_kernel(const cv_adamw_entry* __restrict__ table, float* __restrict__ out) {
    const cv_adamw_entry e = table[blockIdx.y];
    const size_t n = (size_t)e.n, n8 = n / 8;
    if ((size_t)blockIdx.x * 256 >= n8 + 1) return;
    const __nv_bfloat16* x = static_cast<const __nv_bfloat16*>(e.grad);
    float s = 0.f;
    for (size_t i = blockIdx.x * (size_t)256 + threadIdx.x; i < n8; i += (size_t)gridDim.x * 256) {
        uint4 u = reinterpret_cast<const uint4*>(x)[i];
        const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float a = __low2float(p[t]), b = __high2float(p[t]);
            s += a * a + b * b;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 7)) {
        const float a = __bfloat162float(x[n8 * 8 + threadIdx.x]);
        s += a * a;
    }
    s = warp_sum(s);
    __shared__ float sh[8];
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        float t = sh[threadIdx.x];
        t += __shfl_xor_sync(0xffu, t, 4);
        t += __shfl_xor_sync(0xffu, t, 2);
        t += __shfl_xor_sync(0xffu, t, 1);
        if (threadIdx.x == 0) atomicAdd(out, t);
    }
}

}  // namespace

extern "C" int cv_clip_coef(const float* sumsq, float max_norm, float* coef, float* norm_out, int* state,
                            void* stream) {
    CV_REQUIRE(sumsq && coef, "null pointer");
    clip_coef_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(sumsq, max_norm, coef, norm_out, state);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_adamw_step_multi(const cv_adamw_entry* table_dev, int count, float beta1, float beta2, float eps,
                                   const float* grad_scale_dev, float grad_scale, const int* state, void* stream) {
    CV_REQUIRE(table_dev && count > 0 && count <= 65535, "bad table");
    adamw_multi_kernel<<<dim3(MT_CTAS, count), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        table_dev, beta1, beta2, eps, grad_scale_dev, grad_scale, state);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_sumsq_bf16_multi(const cv_adamw_entry* table_dev, int count, float* out, void* stream) {
    CV_REQUIRE(table_dev && out && count > 0 && count <= 65535, "bad table");
    sumsq_multi_kernel<<<dim3(MT_CTAS, count), 256, 0, static_cast<cudaStream_t>(stream)>>>(table_dev, out);
    CV_LAUNCH_CHECK();
    return 0;
}
