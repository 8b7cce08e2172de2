// VQ-VAE training kernels (vqvae/vqvae_zc.py in train() mode), NHWC bf16 activations.
//
//   cv_conv_k4s2_wgrad     weight gradient of nn.Conv2d(k4, s2, p1) and of nn.ConvTranspose2d(k4, s2, p1)
//                          (Encoder :121-129, Decoder :172-191)
//   cv_relu_mask_bf16      dx *= (act > 0): the ReLU backward on a data gradient, from the saved ReLU output
//   cv_conv1x1_out3_bwd    backward of the Decoder's last 1x1 conv 512 -> 3 (:191): masked data gradient, dW, db
//   cv_vq_ema_stats        embed_onehot_sum and embed_sum = flatten^T . onehot of Quantize.forward_ (:68-69)
//
// Every reduction here runs in a fixed order, so equal inputs give equal bits: split-K partials and per-block
// partials go to a workspace and are summed in index order by a second kernel; no floating-point atomics.
//
// Weight gradient.  Both layer types share one form.  With the "small" map S [B, h, w, M] and the "big" map
// G [B, 2h, 2w, N],
//     out[m, n, ky, kx] = sum over (b, y, x) of S[b, y, x, m] * G[b, 2y - 1 + ky, 2x - 1 + kx, n]
// (zero outside G).  Conv2d:          S = dY (M = Cout), G = X (N = Cin)  -> dW in the [Cout, Cin, 4, 4] layout.
//                    ConvTranspose2d: S = X (M = Cin),  G = dY (N = Cout) -> dW in the [Cin, Cout, 4, 4] layout.
// It is a GEMM per tap with K = the B h w pixels and both operands pixel-major (MN-major).  One CTA computes a
// 128 (m) x 256 (n) tile of one tap over one K split: cp.async gathers 32-pixel slices of S and of the tap's
// strided G pixels into a 4-stage shared-memory ring (zero-fill for the padding halo and the K tail), and eight
// warps (2 x 4, 64 x 64 each) run mma.sync m16n8k16 on ldmatrix.trans fragments.  The gather is per 16-byte
// channel chunk, so every tap of every tile shape is handled the same way (no TMA box limits on the map width).
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;                         // 0: zero-fill the 16 bytes
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float* d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ------------------------------------------------------------------------------------------------
// weight gradient of the k4 s2 p1 convolutions
// ------------------------------------------------------------------------------------------------
constexpr int WG_BM = 128;      // tile rows: channels of S
constexpr int WG_BN = 256;      // tile columns: channels of G
constexpr int WG_BK = 32;       // pixels per pipeline stage
constexpr int WG_STAGES = 4;
constexpr int WG_THREADS = 256;
constexpr int WG_S_BYTES = WG_BK * WG_BM * 2;     // 8 KB: 32 pixel rows of 256 B
constexpr int WG_G_BYTES = WG_BK * WG_BN * 2;     // 16 KB: 32 pixel rows of 512 B
constexpr int WG_STAGE_BYTES = WG_S_BYTES + WG_G_BYTES;
constexpr int WG_SMEM_BYTES = WG_STAGES * WG_STAGE_BYTES;

struct WgradParams {
    const __nv_bfloat16* S;   // [B, h, w, M]
    const __nv_bfloat16* G;   // [B, 2h, 2w, N]
    float* part;              // [splits, 16, M, N]
    int h, w, M, N;
    int64_t P;                // B h w
    int64_t k_per_split;      // multiple of WG_BK
};

// byte offset of 16-byte chunk c of pixel row r (row_bytes per row); the XOR on the low three chunk bits puts the
// 8 rows one ldmatrix phase reads on 8 different bank groups
__device__ __forceinline__ uint32_t wg_swz(int r, int c, int row_bytes) {
    return (uint32_t)(r * row_bytes + ((c ^ (r & 7)) << 4));
}

__global__ void __launch_bounds__(WG_THREADS, 1)
conv_wgrad_kernel(const WgradParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int n0 = blockIdx.x * WG_BN;
    const int m0 = blockIdx.y * WG_BM;
    const int tap = blockIdx.z & 15, split = blockIdx.z >> 4;
    const int ky = tap >> 2, kx = tap & 3;
    const int64_t kbeg = split * p.k_per_split;
    const int64_t kend = min(p.P, kbeg + p.k_per_split);
    const int nsteps = (int)((kend - kbeg + WG_BK - 1) / WG_BK);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 2, wn = warp & 3;          // warp tile: rows 64 wm .., columns 64 wn ..
    const int hw = p.h * p.w, GW = 2 * p.w, GH = 2 * p.h;
    const uint32_t sbase = smem_u32(smem);

    // loader roles: S has 32 rows x 16 chunks (2 per thread), G 32 rows x 32 chunks (4 per thread)
    auto load_stage = [&](int step, int slot) {
        const uint32_t sS = sbase + slot * WG_STAGE_BYTES, sG = sS + WG_S_BYTES;
        const int64_t k0 = kbeg + (int64_t)step * WG_BK;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int idx = tid + i * WG_THREADS, r = idx >> 4, c = idx & 15;
            const int64_t px = k0 + r;
            const bool ok = px < kend;
            const __nv_bfloat16* src = p.S + (ok ? px : 0) * p.M + m0 + c * 8;
            cp_async16(sS + wg_swz(r, c, WG_BM * 2), src, ok);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * WG_THREADS, r = idx >> 5, c = idx & 31;
            const int64_t px = k0 + r;
            bool ok = px < kend;
            int64_t goff = 0;
            if (ok) {
                const int64_t b = px / hw;
                const int rem = (int)(px - b * hw);
                const int y = rem / p.w, x = rem - y * p.w;
                const int gy = 2 * y - 1 + ky, gx = 2 * x - 1 + kx;
                ok = gy >= 0 && gy < GH && gx >= 0 && gx < GW;
                goff = ((b * GH + gy) * GW + gx) * p.N;
            }
            const __nv_bfloat16* src = p.G + (ok ? goff : 0) + n0 + c * 8;
            cp_async16(sG + wg_swz(r, c, WG_BN * 2), src, ok);
        }
    };

    float acc[4][8][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
    for (int s = 0; s < WG_STAGES - 1; ++s) {
        if (s < nsteps) load_stage(s, s);
        cp_async_commit();
    }
    // ldmatrix.trans lane roles.  A (m x k, from S rows = k): matrix q = lane / 8 covers k rows 8 (q >> 1) ..,
    // m columns 8 (q & 1) ..  B (k x n, from G rows = k): matrix q covers k rows 8 (q & 1) .., n columns 8 (q >> 1) ..
    const int q = lane >> 3, lr = lane & 7;
    const int a_krow = lr + 8 * (q >> 1), a_mchunk = (wm * 64) / 8 + (q & 1);
    const int b_krow = lr + 8 * (q & 1), b_nchunk = (wn * 64) / 8 + (q >> 1);

    for (int step = 0; step < nsteps; ++step) {
        cp_async_wait<WG_STAGES - 2>();
        __syncthreads();
        {   // refill the slot consumed one iteration ago
            const int nxt = step + WG_STAGES - 1;
            if (nxt < nsteps) load_stage(nxt, nxt % WG_STAGES);
            cp_async_commit();
        }
        const int slot = step % WG_STAGES;
        const uint32_t sS = sbase + slot * WG_STAGE_BYTES, sG = sS + WG_S_BYTES;
#pragma unroll
        for (int kk = 0; kk < WG_BK / 16; ++kk) {
            uint32_t a[4][4], b[8][2];
#pragma unroll
            for (int i = 0; i < 4; ++i)
                ldsm_x4_t(sS + wg_swz(16 * kk + a_krow, a_mchunk + 2 * i, WG_BM * 2), a[i][0], a[i][1], a[i][2], a[i][3]);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                ldsm_x4_t(sG + wg_swz(16 * kk + b_krow, b_nchunk + 2 * j, WG_BN * 2), b[2 * j][0], b[2 * j][1],
                          b[2 * j + 1][0], b[2 * j + 1][1]);
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) mma16816(acc[i][j], a[i], b[j][0], b[j][1]);
        }
    }
    cp_async_wait<0>();

    float* out = p.part + ((size_t)split * 16 + tap) * p.M * p.N;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = m0 + wm * 64 + 16 * i + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = n0 + wn * 64 + 8 * j + 2 * (lane & 3);
            *reinterpret_cast<float2*>(out + (size_t)r * p.N + c) = make_float2(acc[i][j][0], acc[i][j][1]);
            *reinterpret_cast<float2*>(out + (size_t)(r + 8) * p.N + c) = make_float2(acc[i][j][2], acc[i][j][3]);
        }
    }
}

// out[m, n, tap] = sum over splits (in order) of part[s, tap, m, n]
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int splits, int M, int N) {
    const size_t per = (size_t)16 * M * N;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < per; i += (size_t)gridDim.x * blockDim.x) {
        const int tap = (int)(i / ((size_t)M * N));
        const size_t mn = i - (size_t)tap * M * N;
        float s = 0.f;
        for (int k = 0; k < splits; ++k) s += part[k * per + i];
        out[mn * 16 + tap] = s;
    }
}

int wgrad_splits(int64_t P, int M, int N) {
    // enough CTAs for about four per SM, with at least 1024 pixels (32 pipeline steps) per split
    const int64_t ctas = (int64_t)16 * (M / WG_BM) * (N / WG_BN);
    int64_t s = (4LL * cvh::num_sms() + ctas - 1) / ctas;
    const int64_t by_k = P / 1024;
    if (s > by_k) s = by_k;
    if (s < 1) s = 1;
    if (s > 32) s = 32;
    return (int)s;
}

// ------------------------------------------------------------------------------------------------
// ReLU backward from the saved ReLU output
// ------------------------------------------------------------------------------------------------
__global__ void relu_mask_kernel(uint4* __restrict__ dx, const uint4* __restrict__ act, size_t n8) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
        uint4 d = dx[i];
        const uint4 a = act[i];
        uint32_t* dw = reinterpret_cast<uint32_t*>(&d);
        const uint32_t* aw = reinterpret_cast<const uint32_t*>(&a);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // a bf16 is > 0 iff its sign bit is clear and it is not +0 (ReLU outputs are never NaN)
            const uint32_t lo = aw[k] & 0xFFFFu, hi = aw[k] >> 16;
            const uint32_t keep = ((lo != 0 && !(lo & 0x8000u)) ? 0xFFFFu : 0u) |
                                  ((hi != 0 && !(hi & 0x8000u)) ? 0xFFFF0000u : 0u);
            dw[k] &= keep;
        }
        dx[i] = d;
    }
}

// ------------------------------------------------------------------------------------------------
// backward of the decoder's last 1x1 conv (Cin -> 3), one read of the Cin-channel activation
// ------------------------------------------------------------------------------------------------
constexpr int C3_THREADS = 256;
constexpr int C3_MAX_BLOCKS = 1024;

// thread = (pixel lane j, 8-channel group g); block partials part[block][3 * cin + 3] (dW rows then db)
__global__ void __launch_bounds__(C3_THREADS)
conv1x1_out3_bwd_kernel(const float* __restrict__ dr /*[B, 3, H, W]*/, const __nv_bfloat16* __restrict__ x,
                        const float* __restrict__ w /*[3, cin]*/, __nv_bfloat16* __restrict__ dx,
                        float* __restrict__ part, int64_t npix, int hw, int cin) {
    extern __shared__ float red[];                       // [lanes][3 * cin + 3]
    const int groups = cin / 8, lanes = C3_THREADS / groups;
    const int g = threadIdx.x % groups, j = threadIdx.x / groups;
    const int width = 3 * cin + 3;
    float wv[3][8], dw[3][8], db[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int k = 0; k < 8; ++k) { wv[c][k] = w[c * cin + 8 * g + k]; dw[c][k] = 0.f; }
    for (int64_t px = (int64_t)blockIdx.x * lanes + j; px < npix; px += (int64_t)gridDim.x * lanes) {
        const int64_t b = px / hw;
        const int64_t o = px - b * hw;
        float d[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) { d[c] = dr[(b * 3 + c) * hw + o]; db[c] += d[c]; }
        const uint4 xv = *reinterpret_cast<const uint4*>(x + px * cin + 8 * g);
        const __nv_bfloat16* xe = reinterpret_cast<const __nv_bfloat16*>(&xv);
        uint4 ov;
        uint32_t* ow = reinterpret_cast<uint32_t*>(&ov);
#pragma unroll
        for (int k = 0; k < 8; k += 2) {
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float xf = __bfloat162float(xe[k + e]);
#pragma unroll
                for (int c = 0; c < 3; ++c) dw[c][k + e] += d[c] * xf;
                const float s = d[0] * wv[0][k + e] + d[1] * wv[1][k + e] + d[2] * wv[2][k + e];
                v[e] = xf > 0.f ? s : 0.f;
            }
            ow[k / 2] = pack_bf16x2(v[0], v[1]);
        }
        *reinterpret_cast<uint4*>(dx + px * cin + 8 * g) = ov;
    }
    float* mine = red + j * width;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int k = 0; k < 8; ++k) mine[c * cin + 8 * g + k] = dw[c][k];
    if (g == 0) { mine[3 * cin] = db[0]; mine[3 * cin + 1] = db[1]; mine[3 * cin + 2] = db[2]; }
    __syncthreads();
    for (int i = threadIdx.x; i < width; i += C3_THREADS) {
        float s = 0.f;
        for (int l = 0; l < lanes; ++l) s += red[l * width + i];
        part[(size_t)blockIdx.x * width + i] = s;
    }
}

__global__ void block_partials_sum_kernel(const float* __restrict__ part, int blocks, int width,
                                          float* __restrict__ dw, float* __restrict__ db, int ndw) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < width; i += gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < blocks; ++k) s += part[(size_t)k * width + i];
        if (i < ndw) dw[i] = s; else db[i - ndw] = s;
    }
}

// ------------------------------------------------------------------------------------------------
// EMA codebook statistics: each block owns EMA_CODES codes, walks all rows in order and adds the rows whose code
// it owns, so every code's sum is taken in row order
// ------------------------------------------------------------------------------------------------
constexpr int EMA_CODES = 64;
constexpr int EMA_THREADS = 256;

__global__ void __launch_bounds__(EMA_THREADS)
vq_ema_stats_kernel(const int64_t* __restrict__ idx, const float* __restrict__ z, int64_t rows, int dim, int n_embed,
                    float* __restrict__ counts, float* __restrict__ embed_sum /*[dim, n_embed]*/) {
    extern __shared__ float acc[];                       // [EMA_CODES][dim + 1]
    __shared__ int list_row[EMA_THREADS];
    __shared__ uint8_t list_code[EMA_THREADS];
    __shared__ int warp_cnt[EMA_THREADS / 32];
    __shared__ int cnt[EMA_CODES];
    const int c0 = blockIdx.x * EMA_CODES;
    const int ld = dim + 1;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < EMA_CODES * ld; i += EMA_THREADS) acc[i] = 0.f;
    if (tid < EMA_CODES) cnt[tid] = 0;
    __syncthreads();
    for (int64_t r0 = 0; r0 < rows; r0 += EMA_THREADS) {
        const int64_t r = r0 + tid;
        const int64_t code = r < rows ? idx[r] : -1;
        const bool mine = code >= c0 && code < c0 + EMA_CODES;
        const uint32_t ball = __ballot_sync(0xffffffffu, mine);
        if (lane == 0) warp_cnt[warp] = __popc(ball);
        __syncthreads();
        int base = 0, total = 0;
#pragma unroll
        for (int w = 0; w < EMA_THREADS / 32; ++w) { base += w < warp ? warp_cnt[w] : 0; total += warp_cnt[w]; }
        if (mine) {
            const int pos = base + __popc(ball & ((1u << lane) - 1u));
            list_row[pos] = (int)(r - r0);
            list_code[pos] = (uint8_t)(code - c0);
        }
        __syncthreads();
        for (int e = 0; e < total; ++e) {
            const int cl = list_code[e];
            const float* zr = z + (r0 + list_row[e]) * dim;
            for (int d = tid; d < dim; d += EMA_THREADS) acc[cl * ld + d] += zr[d];
            if (tid == 0) cnt[cl] += 1;
        }
        __syncthreads();
    }
    const int ncodes = min(EMA_CODES, n_embed - c0);
    if (tid < ncodes) counts[c0 + tid] = (float)cnt[tid];
    for (int i = tid; i < EMA_CODES * dim; i += EMA_THREADS) {
        const int cl = i % EMA_CODES, d = i / EMA_CODES;
        if (cl < ncodes) embed_sum[(size_t)d * n_embed + c0 + cl] = acc[cl * ld + d];
    }
}

int grid_for(size_t work_items, int threads) {
    size_t blocks = (work_items + threads - 1) / threads;
    size_t cap = (size_t)cvh::num_sms() * 8;
    return (int)(blocks < cap ? (blocks ? blocks : 1) : cap);
}

}  // namespace

extern "C" int64_t cv_conv_k4s2_wgrad_workspace_bytes(int B, int h, int w, int M, int N) {
    const int64_t P = (int64_t)B * h * w;
    return (int64_t)wgrad_splits(P, M, N) * 16 * M * N * (int64_t)sizeof(float);
}

extern "C" int cv_conv_k4s2_wgrad(const void* S, const void* G, float* out, float* workspace, int B, int h, int w,
                                  int M, int N, void* stream) {
    CV_REQUIRE(S && G && out && workspace, "null pointer");
    CV_REQUIRE(B > 0 && h > 0 && w > 0, "map dims must be positive");
    CV_REQUIRE(M % WG_BM == 0 && N % WG_BN == 0, "S channels must be a multiple of 128 and G channels of 256");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(S) & 15) == 0 && (reinterpret_cast<uintptr_t>(G) & 15) == 0,
               "S and G must be 16-byte aligned");
    WgradParams p;
    p.S = static_cast<const __nv_bfloat16*>(S);
    p.G = static_cast<const __nv_bfloat16*>(G);
    p.part = workspace;
    p.h = h; p.w = w; p.M = M; p.N = N;
    p.P = (int64_t)B * h * w;
    const int splits = wgrad_splits(p.P, M, N);
    p.k_per_split = ((p.P + splits - 1) / splits + WG_BK - 1) / WG_BK * WG_BK;
    const int used = (int)((p.P + p.k_per_split - 1) / p.k_per_split);   // every launched split has pixels
    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM_BYTES));
        attr_set = true;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid(N / WG_BN, M / WG_BM, 16 * used);
    conv_wgrad_kernel<<<grid, WG_THREADS, WG_SMEM_BYTES, s>>>(p);
    CV_LAUNCH_CHECK();
    const size_t per = (size_t)16 * M * N;
    wgrad_reduce_kernel<<<grid_for(per, 256), 256, 0, s>>>(workspace, out, used, M, N);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_relu_mask_bf16(void* dx, const void* act, int64_t n, void* stream) {
    CV_REQUIRE(dx && act, "null pointer");
    CV_REQUIRE(n > 0 && n % 8 == 0, "element count must be a positive multiple of 8");
    CV_REQUIRE((reinterpret_cast<uintptr_t>(dx) & 15) == 0 && (reinterpret_cast<uintptr_t>(act) & 15) == 0,
               "dx and act must be 16-byte aligned");
    const size_t n8 = (size_t)n / 8;
    relu_mask_kernel<<<grid_for(n8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<uint4*>(dx), static_cast<const uint4*>(act), n8);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int64_t cv_conv1x1_out3_bwd_workspace_bytes(int cin) {
    return (int64_t)C3_MAX_BLOCKS * (3 * cin + 3) * (int64_t)sizeof(float);
}

extern "C" int cv_conv1x1_out3_bwd(const float* dr, const void* x, const float* w, void* dx, float* dw, float* db,
                                   float* workspace, int B, int H, int W, int cin, void* stream) {
    CV_REQUIRE(dr && x && w && dx && dw && db && workspace, "null pointer");
    CV_REQUIRE(B > 0 && H > 0 && W > 0, "map dims must be positive");
    CV_REQUIRE(cin % 8 == 0 && cin / 8 <= C3_THREADS && C3_THREADS % (cin / 8) == 0,
               "cin must be 8 times a divisor of 256");
    const int64_t npix = (int64_t)B * H * W;
    const int lanes = C3_THREADS / (cin / 8);
    int64_t blocks = (npix + 16 * lanes - 1) / (16 * lanes);       // at least 16 pixels per lane
    if (blocks > C3_MAX_BLOCKS) blocks = C3_MAX_BLOCKS;
    const int width = 3 * cin + 3;
    const size_t smem = (size_t)lanes * width * sizeof(float);
    CV_REQUIRE(smem <= 48 * 1024, "cin too large for the block reduction");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    conv1x1_out3_bwd_kernel<<<(int)blocks, C3_THREADS, smem, s>>>(dr, static_cast<const __nv_bfloat16*>(x), w,
                                                                  static_cast<__nv_bfloat16*>(dx), workspace, npix,
                                                                  H * W, cin);
    CV_LAUNCH_CHECK();
    block_partials_sum_kernel<<<(width + 255) / 256, 256, 0, s>>>(workspace, (int)blocks, width, dw, db, 3 * cin);
    CV_LAUNCH_CHECK();
    return 0;
}

extern "C" int cv_vq_ema_stats(const int64_t* idx, const float* z, int64_t rows, int dim, int n_embed, float* counts,
                               float* embed_sum, void* stream) {
    CV_REQUIRE(idx && z && counts && embed_sum, "null pointer");
    CV_REQUIRE(rows > 0 && dim > 0 && n_embed > 0, "rows, dim and n_embed must be positive");
    const size_t smem = (size_t)EMA_CODES * (dim + 1) * sizeof(float);
    CV_REQUIRE(smem <= 200 * 1024, "dim too large");
    static size_t attr = 0;
    if (smem > 48 * 1024 && smem > attr) {
        CV_CUDA(cudaFuncSetAttribute(vq_ema_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    vq_ema_stats_kernel<<<(n_embed + EMA_CODES - 1) / EMA_CODES, EMA_THREADS, smem,
                          static_cast<cudaStream_t>(stream)>>>(idx, z, rows, dim, n_embed, counts, embed_sum);
    CV_LAUNCH_CHECK();
    return 0;
}
