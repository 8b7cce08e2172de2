// Micro-benchmark of the decode-step CONSUMER: data already in shared memory (no producer, no HBM): how many KB/us can
// the 16 consumer warps push through ld.shared + mma.sync in the kernel's scheme (two groups of 8 warps on alternate
// 16-row x 1280-col stages, per-tile CTA barrier + reduce)?  Variants isolate LDS, HMMA chain, barrier.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
    return r;
}
__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
constexpr int CPW = 5, PITCH = 2624, XPITCH = 5184, STAGE = 16 * PITCH;
// mode bits: 1 = skip HMMA, 2 = skip LDS of weights, 4 = no per-tile barrier/reduce, 8 = two accumulators, 16 = all 16 warps on every stage (K/16 each... uses CPW 5 on half rows?)
__global__ void __launch_bounds__(544, 1) consume_kernel(int tiles, int mode, float* out) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (warp >= 16) return;
    const int g = lane >> 2, q = lane & 3, grp_w = warp / 8, wg = warp % 8;
    const uint32_t xop = smem_u32(smem), ring = xop + 8 * XPITCH;
    float* part = reinterpret_cast<float*>(smem + 8 * XPITCH + 4 * STAGE);
    float dA[4] = {0, 0, 0, 0}, dB[4] = {0, 0, 0, 0};
    int sq = 0, pbuf = 0;
    float keep = 0.f;
    for (int t = 0; t < tiles; ++t) {
        for (int ks = 0; ks < 2; ++ks) {
            const int st = sq & 3;
            if ((sq & 1) == grp_w) {
                const uint32_t wa = ring + st * STAGE + g * PITCH + (wg * 160 + q * 8) * 2;
                const uint32_t xa = xop + g * XPITCH + (ks * 1280 + wg * 160 + q * 8) * 2;
                uint4 w0[CPW], w1[CPW], xv[CPW];
#pragma unroll
                for (int c = 0; c < CPW; ++c) {
                    if (!(mode & 2)) { w0[c] = lds128(wa + c * 64); w1[c] = lds128(wa + 8 * PITCH + c * 64); }
                    else { w0[c] = make_uint4(c, t, ks, lane); w1[c] = make_uint4(lane, c, t, ks); }
                    xv[c] = g < 4 ? lds128(xa + c * 64) : make_uint4(0, 0, 0, 0);
                }
                if (!(mode & 1)) {
#pragma unroll
                    for (int c = 0; c < CPW; ++c) {
                        if (mode & 8) {
                            mma_16816(dA, w0[c].x, w1[c].x, w0[c].y, w1[c].y, xv[c].x, xv[c].y);
                            mma_16816(dB, w0[c].z, w1[c].z, w0[c].w, w1[c].w, xv[c].z, xv[c].w);
                        } else {
                            mma_16816(dA, w0[c].x, w1[c].x, w0[c].y, w1[c].y, xv[c].x, xv[c].y);
                            mma_16816(dA, w0[c].z, w1[c].z, w0[c].w, w1[c].w, xv[c].z, xv[c].w);
                        }
                    }
                } else {
#pragma unroll
                    for (int c = 0; c < CPW; ++c) dA[0] += __uint_as_float(w0[c].x ^ w1[c].y ^ xv[c].z);
                }
                __syncwarp();
            }
            ++sq;
        }
        if (!(mode & 4)) {
            float* pw = part + ((pbuf * 16 + warp) * 16) * 8;
            pw[g * 8 + 2 * q] = dA[0] + dB[0]; pw[g * 8 + 2 * q + 1] = dA[1] + dB[1];
            pw[(g + 8) * 8 + 2 * q] = dA[2] + dB[2]; pw[(g + 8) * 8 + 2 * q + 1] = dA[3] + dB[3];
            dA[0] = dA[1] = dA[2] = dA[3] = 0.f; dB[0] = dB[1] = dB[2] = dB[3] = 0.f;
            asm volatile("bar.sync 1, 512;" ::: "memory");
            if (tid < 128) {
                const int mi = tid >> 4, nn = tid & 15;
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < 16; ++w) v += part[((pbuf * 16 + w) * 16 + nn) * 8 + mi];
                keep += v;
            }
            pbuf ^= 1;
        }
    }
    if (keep + dA[0] + dB[1] == 123.456f) out[0] = keep;
}
int main() {
    float* out; cudaMalloc(&out, 4);
    const size_t smem = 8 * XPITCH + 4 * STAGE + 16384;
    cudaFuncSetAttribute(consume_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int tiles = 20000;
    const char* names[] = {"full (current scheme)", "no HMMA", "no weight LDS", "no LDS, no HMMA", "no tile barrier", "no HMMA, no barrier",
                           "two accumulators", "two acc, no barrier"};
    const int modes[] = {0, 1, 2, 3, 4, 5, 8, 12};
    for (int i = 0; i < 8; ++i) {
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        consume_kernel<<<132, 544, smem>>>(100, modes[i], out);
        cudaEventRecord(e0);
        consume_kernel<<<132, 544, smem>>>(tiles, modes[i], out);
        cudaEventRecord(e1);
        cudaError_t err = cudaDeviceSynchronize();
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        printf("%-28s %8.3f ms  %6.3f us/tile  %7.1f KB/us per SM  (%s)\n", names[i], ms, ms * 1e3 / tiles,
               2.0 * 16 * 2560 / 1024.0 / (ms * 1e3 / tiles), cudaGetErrorString(err));
    }
    return 0;
}
