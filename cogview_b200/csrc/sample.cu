// Sampling epilogue of the autoregressive loop as one kernel (one CTA per sequence):
//   logits / temperature -> invalid vocabulary slices -> top-k filter -> softmax -> one multinomial draw ->
//   log-probability, token hand-over to the next decode step.
// Reference: generation/sampling.py:157-183 and top_k_logits :24-33 (`logits[logits < kth] = -inf`: every logit equal
// to the k-th largest survives).  The k-th largest value is found exactly with a 4-pass radix select on the
// order-preserving integer image of the floats; the row (<= 233 KB, 32 KB for image tokens) stays in L1/L2.
//
// Nucleus (top-p) filtering, top_k_logits :34-47, is the NUCLEUS instantiation: applied after top-k, over the
// softmax of the top-k survivors.  The reference sorts descending, takes the cumulative sum and shifts it by one, so
// a token survives iff the probability mass strictly above it is <= top_p (the first token that takes the mass past
// top_p is kept).  The boundary key is found with a second 4-pass radix descent on the same keys whose histograms
// hold probability MASS per bin: exp(x - max) in 2^-40 fixed point (<= 2^56 over 58240 entries), summed first over
// the lanes of a warp that share a bin, then with exact integer shared-memory atomics, so the sums do not depend on
// the order of the adds and every call is bit-reproducible.  Every token
// whose logit equals the boundary logit is kept (the same rule as top-k's `logits < kth`); torch.sort leaves the
// order among ties unspecified, so the reference has no defined answer there.  top_p >= 1, or a mass that is never
// exceeded, keeps every top-k survivor.
#include "common.cuh"
#include "host.h"
#include "../../include/cogview_b200.h"

namespace {
using namespace cv;

constexpr int ST = 1024;            // threads per CTA
constexpr int SW = ST / 32;

struct SampleParams {
    const float* logits;
    int64_t ld;
    int V, b, top_k, nv, nvalid;
    float temperature;
    int vlo[4], vhi[4];
    uint64_t seed;
    const uint64_t* seed_dev;
    int64_t* step;
    int64_t* next_ids;
    int64_t* out_tokens;
    int64_t ld_out;
    float* score_acc;
    int64_t* pos;
    int* cur_len;
    unsigned int* done;
    float* probs_out;
};

__device__ __forceinline__ uint32_t f2key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <bool NUCLEUS>
__global__ void __launch_bounds__(ST) sample_topk_kernel(const SampleParams p, const float top_p) {
    __shared__ int hist[256];
    __shared__ float wred[SW];
    __shared__ float wcum[SW];
    __shared__ uint32_t s_prefix;
    __shared__ int s_krem, s_warp, s_token;
    __shared__ float s_total, s_psel;
    const int row = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* lg = p.logits + (size_t)row * p.ld;
    const int64_t stepval = p.step ? *p.step : 0;
    const int R = ((p.nvalid + ST - 1) / ST) * 32;      // virtual indices per warp (multiple of 32)
    const int nit = R / 32;
    auto real_index = [&](int i) -> int {
        int idx = -1;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            if (r < p.nv && idx < 0) {
                const int len = p.vhi[r] - p.vlo[r];
                if (i < len) idx = p.vlo[r] + i;
                else i -= len;
            }
        }
        return idx;
    };
    auto value = [&](int idx) -> float { return lg[idx] / p.temperature; };

    // ---- maximum over the valid entries -----------------------------------------------------------
    float mx = -INFINITY;
    for (int it = 0; it < nit; ++it) {
        const int i = warp * R + it * 32 + lane;
        if (i < p.nvalid) mx = fmaxf(mx, value(real_index(i)));
    }
    mx = warp_max(mx);
    if (lane == 0) wred[warp] = mx;
    __syncthreads();
    mx = wred[0];
#pragma unroll
    for (int w = 1; w < SW; ++w) mx = fmaxf(mx, wred[w]);
    __syncthreads();

    // ---- exact k-th largest key ---------------------------------------------------------------------
    uint32_t thr = 0;                                   // keep key >= thr
    if (p.top_k > 0 && p.top_k < p.nvalid) {
        if (tid == 0) { s_prefix = 0; s_krem = p.top_k; }
        uint32_t himask = 0;
        for (int shift = 24; shift >= 0; shift -= 8) {
            if (tid < 256) hist[tid] = 0;
            __syncthreads();
            const uint32_t prefix = s_prefix;
            for (int it = 0; it < nit; ++it) {
                const int i = warp * R + it * 32 + lane;
                if (i < p.nvalid) {
                    const uint32_t key = f2key(value(real_index(i)));
                    if (((key ^ prefix) & himask) == 0) atomicAdd(&hist[(key >> shift) & 255], 1);
                }
            }
            __syncthreads();
            if (warp == 0) {
                // lane L owns bins 255-8L .. 248-8L (descending); find the bin where the count from the top reaches k
                int c = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) c += hist[255 - 8 * lane - j];
                int cum = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, cum, o);
                    if (lane >= o) cum += t;
                }
                const int krem = s_krem;
                const unsigned int bal = __ballot_sync(0xffffffffu, cum >= krem);
                const int sel = __ffs(bal) - 1;             // bal != 0: the pass covers >= krem elements
                if (lane == sel) {
                    int before = cum - c;
                    for (int j = 0; j < 8; ++j) {
                        const int bin = 255 - 8 * lane - j;
                        const int hcnt = hist[bin];
                        if (before + hcnt >= krem) {
                            s_prefix = prefix | ((uint32_t)bin << shift);
                            s_krem = krem - before;
                            break;
                        }
                        before += hcnt;
                    }
                }
            }
            himask |= 0xffu << shift;
            __syncthreads();
        }
        thr = s_prefix;
    }

    if constexpr (NUCLEUS) {
        // ---- nucleus boundary: the largest key whose mass strictly above is > limit ends the kept set ----------
        // The mass of a bin is kept as three 16-bit digits in 32-bit counters: every add is < 2^16 per digit and a
        // bin gets at most 58240 adds, so the counters never wrap, and 32-bit shared atomics are native (a 64-bit
        // shared add is a compare-and-swap loop, which the few hot bins of the first pass would serialise on).
        __shared__ unsigned int mhist[3][256];
        __shared__ unsigned long long s_above;          // mass of the kept keys above the current prefix
        __shared__ uint32_t s_pprefix;
        __shared__ int s_all;
        auto bin_mass = [&](int bin) -> unsigned long long {
            return (unsigned long long)mhist[0][bin] + ((unsigned long long)mhist[1][bin] << 16) +
                   ((unsigned long long)mhist[2][bin] << 32);
        };
        if (top_p < 1.f) {
            if (tid == 0) { s_pprefix = 0; s_above = 0; s_all = 0; }
            unsigned long long limit = 0;                   // floor(top_p * total), warp 0 only
            uint32_t himask = 0;
            for (int shift = 24; shift >= 0; shift -= 8) {
                if (tid < 256) mhist[0][tid] = mhist[1][tid] = mhist[2][tid] = 0u;
                __syncthreads();
                const uint32_t prefix = s_pprefix;
                for (int it = 0; it < nit; ++it) {
                    const int i = warp * R + it * 32 + lane;
                    unsigned int bin = 256u;                // 256: this lane adds nothing
                    unsigned long long w = 0;               // exp(x - max) * 2^40 <= 2^40
                    if (i < p.nvalid) {
                        const float x = value(real_index(i));
                        const uint32_t key = f2key(x);
                        if (key >= thr && ((key ^ prefix) & himask) == 0) {
                            bin = (key >> shift) & 255u;
                            w = __float2ull_rz(__expf(x - mx) * 0x1p40f);
                        }
                    }
                    if (__any_sync(0xffffffffu, bin < 256u)) {
                        // one add per distinct bin of the warp: the lanes of a bin sum their 20-bit halves
                        const unsigned int peers = __match_any_sync(0xffffffffu, bin);
                        const unsigned int lo = __reduce_add_sync(peers, (unsigned int)(w & 0xfffffu));
                        const unsigned int hi = __reduce_add_sync(peers, (unsigned int)(w >> 20));
                        if (bin < 256u && lane == __ffs(peers) - 1) {
                            const unsigned long long s = ((unsigned long long)hi << 20) + lo;     // <= 2^45
                            atomicAdd(&mhist[0][bin], (unsigned int)(s & 0xffffu));
                            atomicAdd(&mhist[1][bin], (unsigned int)((s >> 16) & 0xffffu));
                            atomicAdd(&mhist[2][bin], (unsigned int)(s >> 32));
                        }
                    }
                }
                __syncthreads();
                if (warp == 0) {
                    // lane L owns bins 255-8L .. 248-8L (descending); find the bin where the mass from the top
                    // passes the limit
                    unsigned long long c = 0;
#pragma unroll
                    for (int j = 0; j < 8; ++j) c += bin_mass(255 - 8 * lane - j);
                    unsigned long long cum = c;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned long long t = __shfl_up_sync(0xffffffffu, cum, o);
                        if (lane >= o) cum += t;
                    }
                    if (shift == 24)                        // the first pass holds every kept entry
                        limit = (unsigned long long)((double)top_p * (double)__shfl_sync(0xffffffffu, cum, 31));
                    const unsigned long long above = s_above;
                    const unsigned int bal = __ballot_sync(0xffffffffu, above + cum > limit);
                    const int sel = __ffs(bal) - 1;
                    if (bal == 0) {                         // first pass only: the mass never exceeds top_p
                        if (lane == 0) s_all = 1;
                    } else if (lane == sel) {
                        unsigned long long before = above + cum - c;
                        for (int j = 0; j < 8; ++j) {
                            const int bin = 255 - 8 * lane - j;
                            const unsigned long long m = bin_mass(bin);
                            if (before + m > limit) {
                                s_pprefix = prefix | ((uint32_t)bin << shift);
                                s_above = before;
                                break;
                            }
                            before += m;
                        }
                    }
                }
                himask |= 0xffu << shift;
                __syncthreads();
                if (s_all) break;
            }
            if (!s_all) thr = max(thr, s_pprefix);
        }
    }

    // ---- softmax denominator over the kept entries, in (warp, iteration, lane) order ---------------
    float local = 0.f;
    for (int it = 0; it < nit; ++it) {
        const int i = warp * R + it * 32 + lane;
        if (i < p.nvalid) {
            const float x = value(real_index(i));
            if (f2key(x) >= thr) local += __expf(x - mx);
        }
    }
    local = warp_sum(local);
    if (lane == 0) wred[warp] = local;
    __syncthreads();
    if (tid == 0) {
        float run = 0.f;
        for (int w = 0; w < SW; ++w) { run += wred[w]; wcum[w] = run; }
        s_total = run;
        const uint4 rnd = philox4x32_10(p.seed_dev ? *p.seed_dev : p.seed, (uint64_t)stepval, (uint32_t)row);
        const float u = (float)(rnd.x >> 8) * (1.0f / 16777216.0f) * run;
        int wsel = -1, wlast = 0;
        for (int w = 0; w < SW; ++w) {
            if (wred[w] > 0.f) wlast = w;
            if (wsel < 0 && u < wcum[w] && wred[w] > 0.f) wsel = w;
        }
        s_warp = wsel < 0 ? wlast : wsel;
        s_psel = u;                                     // reused below as the scaled uniform
        s_token = -1;
    }
    __syncthreads();
    const float total = s_total;
    if (warp == s_warp) {
        const float u = s_psel;
        float run = warp == 0 ? 0.f : wcum[warp - 1];
        int chosen = -1, last_kept = -1;
        float pch = 0.f, plast = 0.f;
        for (int it = 0; it < nit && chosen < 0; ++it) {
            const int i = warp * R + it * 32 + lane;
            float e = 0.f;
            int idx = -1;
            if (i < p.nvalid) {
                idx = real_index(i);
                const float x = value(idx);
                if (f2key(x) >= thr) e = __expf(x - mx);
            }
            float inc = e;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            const unsigned int hit = __ballot_sync(0xffffffffu, e > 0.f && u < run + inc);
            const unsigned int kept = __ballot_sync(0xffffffffu, e > 0.f);
            if (hit) {
                const int src = __ffs(hit) - 1;
                chosen = __shfl_sync(0xffffffffu, idx, src);
                pch = __shfl_sync(0xffffffffu, e, src);
            } else if (kept) {
                const int src = 31 - __clz(kept);
                last_kept = __shfl_sync(0xffffffffu, idx, src);
                plast = __shfl_sync(0xffffffffu, e, src);
            }
            run += __shfl_sync(0xffffffffu, inc, 31);
        }
        if (chosen < 0) { chosen = last_kept; pch = plast; }   // rounding at the very end of the CDF
        if (lane == 0) { s_token = chosen; s_psel = pch / total; }
    }
    __syncthreads();

    if (p.probs_out != nullptr) {
        float* po = p.probs_out + (size_t)row * p.ld;
        for (int i = tid; i < p.V; i += ST) po[i] = 0.f;
        __syncthreads();
        for (int it = 0; it < nit; ++it) {
            const int i = warp * R + it * 32 + lane;
            if (i < p.nvalid) {
                const int idx = real_index(i);
                const float x = value(idx);
                if (f2key(x) >= thr) po[idx] = __expf(x - mx) / total;
            }
        }
    }
    if (tid == 0) {
        const int64_t tok = s_token;
        p.next_ids[row] = tok;
        if (p.out_tokens) p.out_tokens[(size_t)row * p.ld_out + stepval] = tok;
        if (p.score_acc) p.score_acc[row] += logf(s_psel);
        if (p.pos) p.pos[row] += 1;
        if (p.done != nullptr) {
            __threadfence();
            const unsigned int old = atomicAdd(p.done, 1u);
            if (old == (unsigned int)(p.b - 1)) {          // every CTA has read *step: advance the shared scalars
                if (p.cur_len) *p.cur_len += 1;
                if (p.step) *p.step += 1;
                *p.done = 0u;
            }
        }
    }
}

}  // namespace

extern "C" int cv_sample_topk(const float* logits, int64_t ld, int b, int vocab, float temperature, int top_k,
                              const int* valid, int n_valid, uint64_t seed, const uint64_t* seed_dev, int64_t* step,
                              int64_t* next_ids, int64_t* out_tokens, int64_t ld_out, float* score_acc, int64_t* pos,
                              int* cur_len, unsigned int* done_counter, float* probs_out, float top_p, void* stream) {
    CV_REQUIRE(logits && next_ids && valid, "null pointer");
    CV_REQUIRE(b >= 1 && vocab >= 1 && ld >= vocab, "bad sizes");
    CV_REQUIRE(n_valid >= 1 && n_valid <= 4, "1..4 valid vocabulary ranges");
    CV_REQUIRE(temperature > 0.f, "temperature must be positive");
    CV_REQUIRE((cur_len == nullptr && step == nullptr) || done_counter != nullptr,
               "done_counter is required when cur_len / step are advanced");
    SampleParams p;
    p.logits = logits; p.ld = ld; p.V = vocab; p.b = b; p.top_k = top_k; p.nv = n_valid;
    p.temperature = temperature;
    int total = 0;
    for (int r = 0; r < 4; ++r) {
        p.vlo[r] = r < n_valid ? valid[2 * r] : 0;
        p.vhi[r] = r < n_valid ? valid[2 * r + 1] : 0;
        if (r < n_valid) {
            CV_REQUIRE(p.vlo[r] >= 0 && p.vhi[r] > p.vlo[r] && p.vhi[r] <= vocab, "valid range out of bounds");
            CV_REQUIRE(r == 0 || p.vlo[r] >= p.vhi[r - 1], "valid ranges must be sorted and disjoint");
            total += p.vhi[r] - p.vlo[r];
        }
    }
    p.nvalid = total;
    p.seed = seed; p.seed_dev = seed_dev; p.step = step; p.next_ids = next_ids; p.out_tokens = out_tokens; p.ld_out = ld_out;
    p.score_acc = score_acc; p.pos = pos; p.cur_len = cur_len; p.done = done_counter; p.probs_out = probs_out;
    if (top_p > 0.f) sample_topk_kernel<true><<<b, ST, 0, static_cast<cudaStream_t>(stream)>>>(p, top_p);
    else sample_topk_kernel<false><<<b, ST, 0, static_cast<cudaStream_t>(stream)>>>(p, 0.f);
    CV_LAUNCH_CHECK();
    return 0;
}
