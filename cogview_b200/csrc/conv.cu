// VQ-VAE convolutions as im2col-free implicit GEMMs on wgmma (NHWC bf16 activations).
//
//   cv_conv2d_k4s2           nn.Conv2d(Cin, Cout, 4, stride=2, padding=1)          encoder, /root/reference/vqvae/vqvae_zc.py:121-129
//   cv_conv_transpose2d_k4s2 nn.ConvTranspose2d(Cin, Cout, 4, stride=2, padding=1) decoder, vqvae/vqvae_zc.py:172-191
//
// GEMM view: rows = output pixels (128 per tile), columns = output channels, K = taps x Cin.  The A tile of one
// tap is one TMA box of the NHWC input — [64 channels x TW x TH x NB] with traversal stride 2 in W and H for the
// strided convolution (elementStrides), out-of-bounds coordinates zero-filled by TMA (that IS the padding) — so
// no im2col buffer is ever materialised.  Weights are pre-packed [tap][Cout][Cin] (K-major B tiles).
// Tile shapes over the [B, H, W] grid of tile pixels (output grid for the strided conv, input grid for a phase):
//   W <= 128, H and W powers of two: whole rows, TW = W, TH = 128 / W (NB = 1), or whole images (NB = 128 / (H W));
//   W > 128, W % 128 == 0, any H:    row segments, TW = 128, TH = NB = 1 (one tile = columns x0 .. x0+127 of
//                                    one row; a TMA box extent is at most 256, so the strided conv's 2 TW and a
//                                    phase's TW cannot cover a wider row).
// The transposed convolution is computed as its 4 sub-pixel phases (each a 2x2-tap stride-1 convolution on the
// input grid); a phase's output pixels are scattered to (2a+py, 2b+px).
// Pipeline and warpgroup roles are those of gemm.cu; epilogue = bias (+ReLU) -> bf16 -> global stores.
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
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

struct ConvParams {
    int Cin, Cout;
    int H, W;            // tile grid: output dims for the strided conv, input dims for a transposed-conv phase
    int TH, NB;          // tile = NB images x TH rows x W columns = 128 pixels (W <= 128)
    int tiles_per_image; // (H*W)/128 when >= 1 (then NB == 1)
    int row_segs;        // W > 128: tiles per row (W / 128; TH = NB = 1); 0 when tiles span whole rows
    int num_m_tiles, num_n_blocks, kc_blocks, ntaps;
    int py, px;          // transposed conv: output phase
    const __nv_bfloat16* bias;
    int relu;
    __nv_bfloat16* y;    // NHWC output
};

template <int N>
__device__ __forceinline__ void conv_mma(float* acc, uint64_t da, uint64_t db, uint32_t sc) {
    if constexpr (N == 256) wgmma_ss_n256<0, 0>(*reinterpret_cast<float(*)[128]>(acc), da, db, sc);
    else wgmma_ss_n128<0, 0>(*reinterpret_cast<float(*)[64]>(acc), da, db, sc);
}

// MODE 1: conv k4 s2 p1.  MODE 2: one phase of convT k4 s2 p1.
template <int BN, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const ConvParams p) {
    using C = Cfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + C::STAGES;          // one arrive per consumer warp

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int num_tiles = p.num_m_tiles * p.num_n_blocks;
    const int num_k_blocks = p.ntaps * p.kc_blocks;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
        for (int i = 0; i < C::STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    auto tile_origin = [&](int mt, int& b0, int& y0, int& x0) {
        x0 = 0;
        if (p.row_segs > 0) {
            const int t = mt % p.tiles_per_image;
            b0 = mt / p.tiles_per_image; y0 = t / p.row_segs; x0 = (t % p.row_segs) * BM;
        } else if (p.tiles_per_image >= 1) { b0 = mt / p.tiles_per_image; y0 = (mt % p.tiles_per_image) * p.TH; }
        else { b0 = mt * p.NB; y0 = 0; }
    };

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tid == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int mt = tile % p.num_m_tiles;
                const int n0 = (tile / p.num_m_tiles) * BN;
                int b0, y0, x0;
                tile_origin(mt, b0, y0, x0);
                for (int kb = 0; kb < num_k_blocks; ++kb) {
                    const int tap = kb / p.kc_blocks, kc = kb - tap * p.kc_blocks;
                    int ax, ay, wtap;
                    if (MODE == 1) {
                        const int ky = tap >> 2, kx = tap & 3;
                        ax = 2 * x0 - 1 + kx;
                        ay = 2 * y0 - 1 + ky;
                        wtap = tap;
                    } else {
                        const int ty = tap >> 1, tx = tap & 1;
                        // output parity 0 uses kernel rows {1,3} at input offsets {0,-1}; parity 1 uses {0,2} at {+1,0}
                        const int ky = p.py == 0 ? (ty == 0 ? 1 : 3) : (ty == 0 ? 0 : 2);
                        const int kx = p.px == 0 ? (tx == 0 ? 1 : 3) : (tx == 0 ? 0 : 2);
                        const int dy = p.py == 0 ? (ty == 0 ? 0 : -1) : (ty == 0 ? 1 : 0);
                        const int dx = p.px == 0 ? (tx == 0 ? 0 : -1) : (tx == 0 ? 1 : 0);
                        ax = x0 + dx;
                        ay = y0 + dy;
                        wtap = ky * 4 + kx;
                    }
                    mbar_wait<false>(&empty_bar[stage], phase ^ 1);
                    uint8_t* sA = smem + stage * C::STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], C::STAGE_BYTES);
                    tma_load_4d(sA, &tmA, &full_bar[stage], kc * BK, ax, ay, b0);
                    tma_load_2d(sA + C::A_BYTES, &tmB, &full_bar[stage], kc * BK, wtap * p.Cout + n0);
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        setmaxnreg_inc<232>();
        const int half = wg - 1;
        const int warp = tid >> 5, lane = tid & 31;
        const int r_in = 64 * half + 16 * warp + (lane >> 2);   // this thread's pixels r_in, r_in + 8 of the tile
        const int c_in = 2 * (lane & 3);
        int stage = 0; uint32_t phase = 0;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int mt = tile % p.num_m_tiles;
            const int n0 = (tile / p.num_m_tiles) * BN;
            int prev = -1;
            for (int kb = 0; kb < num_k_blocks; ++kb) {
                mbar_wait<false>(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem + stage * C::STAGE_BYTES) + half * (64 * 128);
                const uint32_t b_addr = smem_u32(smem + stage * C::STAGE_BYTES + C::A_BYTES);
                fence_regs(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k)
                    conv_mma<BN>(acc, make_smem_desc_sw128(a_addr + k * 32, 0, 1024),
                                 make_smem_desc_sw128(b_addr + k * 32, 0, 1024), (kb | k) != 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<1>();
                if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
                prev = stage;
                if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            int b0, y0, x0;
            tile_origin(mt, b0, y0, x0);
            size_t out_row[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r_in + 8 * h;
                if (MODE == 1) {   // tiles are consecutive 128-pixel runs of the NHWC output in every tiling
                    out_row[h] = (size_t)mt * BM + r;
                } else {   // tile row r = x + W * j, j = (image - b0) * TH + (row - y0) on the input grid
                           // (row segments: j = 0, x = r, input column x0 + r)
                    const int j = r / p.W, x = r % p.W;
                    out_row[h] = ((size_t)2 * (b0 * p.H + y0 + j) + p.py) * (2 * p.W) + 2 * (x0 + x) + p.px;
                }
            }
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
                const int col = n0 + 8 * i + c_in;
                float b0f = 0.f, b1f = 0.f;
                if (p.bias != nullptr) { b0f = __bfloat162float(p.bias[col]); b1f = __bfloat162float(p.bias[col + 1]); }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float v0 = acc[4 * i + 2 * h] + b0f, v1 = acc[4 * i + 2 * h + 1] + b1f;
                    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    *reinterpret_cast<uint32_t*>(p.y + out_row[h] * p.Cout + col) = pack_bf16x2(v0, v1);
                }
            }
        }
    }
}

bool pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }

template <int BN, int MODE>
int launch_conv(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvParams& p, cudaStream_t s) {
    auto kern = conv_kernel<BN, MODE>;
    static bool attr_set = false;
    if (!attr_set) {
        CV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM_BYTES));
        attr_set = true;
    }
    const int tiles = p.num_m_tiles * p.num_n_blocks;
    const int grid = tiles < cvh::num_sms() ? tiles : cvh::num_sms();
    kern<<<grid, NUM_THREADS, Cfg<BN>::SMEM_BYTES, s>>>(tmA, tmB, p);
    CV_LAUNCH_CHECK();
    return 0;
}

// fills the tile decomposition for a [B, H, W] pixel grid; returns false if it cannot be tiled by 128
bool plan_tiles(int B, int H, int W, ConvParams& p) {
    if (W > BM) {   // row segments
        if (W % BM != 0 || H < 1) return false;
        p.H = H; p.W = W;
        p.NB = 1; p.TH = 1; p.row_segs = W / BM; p.tiles_per_image = H * p.row_segs;
        p.num_m_tiles = B * p.tiles_per_image;
        return true;
    }
    if (!pow2(W) || !pow2(H)) return false;
    p.H = H; p.W = W;
    if (H * W >= 128) {
        p.NB = 1; p.TH = 128 / W; p.tiles_per_image = (H * W) / 128;
        p.num_m_tiles = B * p.tiles_per_image;
    } else {
        p.NB = 128 / (H * W); p.TH = H; p.tiles_per_image = 0;
        if (B % p.NB != 0) return false;
        p.num_m_tiles = B / p.NB;
    }
    return true;
}

}  // namespace

extern "C" int cv_conv2d_k4s2(const void* x, const void* w_packed, const void* bias, void* y, int B, int IH, int IW,
                              int Cin, int Cout, int relu, void* stream) {
    CV_REQUIRE(x && w_packed && y, "null pointer");
    CV_REQUIRE(Cin % 64 == 0 && Cout % 128 == 0, "Cin must be a multiple of 64 and Cout of 128");
    CV_REQUIRE(IH % 2 == 0 && IW % 2 == 0, "input height/width must be even");
    const int OH = IH / 2, OW = IW / 2;
    ConvParams p = {};
    CV_REQUIRE(plan_tiles(B, OH, OW, p), "output W must be a power of two <= 128 (with H a power of two and 128 pixels "
                                         "tiling the batch) or a multiple of 128");
    p.Cin = Cin; p.Cout = Cout; p.kc_blocks = Cin / 64; p.ntaps = 16; p.bias = static_cast<const __nv_bfloat16*>(bias);
    p.relu = relu;
    const int BN = (Cout % 256 == 0) ? 256 : 128;
    p.num_n_blocks = Cout / BN;
    p.y = static_cast<__nv_bfloat16*>(y);
    alignas(64) CUtensorMap tmA, tmB;
    {   // input NHWC as [C, W, H, B], traversal stride 2 in W and H
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)IW, (uint64_t)IH, (uint64_t)B};
        uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)IW * Cin * 2, (uint64_t)IH * IW * Cin * 2};
        uint32_t es[4] = {1, 2, 2, 1};
        int rc;
        if (p.row_segs > 0) {   // 128 output columns of one output row
            uint32_t box[4] = {64, (uint32_t)(2 * BM), 2, 1};
            rc = cvh::encode_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x, dims, str, box, es, cvh::Swizzle::B128);
        } else {
            uint32_t box[4] = {64, (uint32_t)(2 * OW), (uint32_t)(2 * p.TH), (uint32_t)p.NB};
            rc = cvh::encode_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x, dims, str, box, es, cvh::Swizzle::B128);
        }
        if (rc) return rc;
    }
    int rc = cvh::encode_tmap_2d_bf16(&tmB, w_packed, (uint64_t)16 * Cout, Cin, Cin, BN, 64);
    if (rc) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return BN == 256 ? launch_conv<256, 1>(tmA, tmB, p, s) : launch_conv<128, 1>(tmA, tmB, p, s);
}

extern "C" int cv_conv_transpose2d_k4s2(const void* x, const void* w_packed, const void* bias, void* y, int B, int IH,
                                        int IW, int Cin, int Cout, int relu, void* stream) {
    CV_REQUIRE(x && w_packed && y, "null pointer");
    CV_REQUIRE(Cin % 64 == 0 && Cout % 128 == 0, "Cin must be a multiple of 64 and Cout of 128");
    ConvParams p = {};
    CV_REQUIRE(plan_tiles(B, IH, IW, p), "input W must be a power of two <= 128 (with H a power of two and 128 pixels "
                                         "tiling the batch) or a multiple of 128");
    p.Cin = Cin; p.Cout = Cout; p.kc_blocks = Cin / 64; p.ntaps = 4; p.bias = static_cast<const __nv_bfloat16*>(bias);
    p.relu = relu;
    const int BN = (Cout % 256 == 0) ? 256 : 128;
    p.num_n_blocks = Cout / BN;
    p.y = static_cast<__nv_bfloat16*>(y);
    alignas(64) CUtensorMap tmA, tmB;
    {   // input NHWC as [C, W, H, B], unit strides; halo taps fall outside and are zero-filled
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)IW, (uint64_t)IH, (uint64_t)B};
        uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)IW * Cin * 2, (uint64_t)IH * IW * Cin * 2};
        int rc;
        if (p.row_segs > 0) {   // 128 input columns of one input row
            uint32_t box[4] = {64, (uint32_t)BM, 1, 1};
            rc = cvh::encode_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x, dims, str, box, nullptr,
                                  cvh::Swizzle::B128);
        } else {
            uint32_t box[4] = {64, (uint32_t)IW, (uint32_t)p.TH, (uint32_t)p.NB};
            rc = cvh::encode_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x, dims, str, box, nullptr,
                                  cvh::Swizzle::B128);
        }
        if (rc) return rc;
    }
    int rc = cvh::encode_tmap_2d_bf16(&tmB, w_packed, (uint64_t)16 * Cout, Cin, Cin, BN, 64);
    if (rc) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    for (int ph = 0; ph < 4; ++ph) {
        p.py = ph >> 1; p.px = ph & 1;
        rc = BN == 256 ? launch_conv<256, 2>(tmA, tmB, p, s) : launch_conv<128, 2>(tmA, tmB, p, s);
        if (rc) return rc;
    }
    return 0;
}
