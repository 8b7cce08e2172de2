// Tile walk of the sparse training attention (mpu/sparse_transformer.py:675-725), shared by the two backward passes, the
// keep-bit generator of its attention-probability dropout and the host that sizes the keep-bit buffer.  attn_fwd_kernel
// computes its walk (jb0, nband, npt) inline with the same expressions as fwd_band_first / fwd_band_count /
// fwd_sees_pivots (with the helpers inlined there, ptxas spills in the dropout instantiation at 168 registers).
#pragma once
#include <stdint.h>

namespace cv {
namespace sparse {

constexpr int TILE = 128;   // query block = key tile = 128 rows (BQ / BKV of the forward, BLK of the backward)

// first band key of query i: max(0, i / w - times + 1) * w
__host__ __device__ __forceinline__ int band_start(int i, int w, int times) {
    const int g = i / w - times + 1;
    return g > 0 ? g * w : 0;
}
__host__ __device__ __forceinline__ int last_query(int qb, int s) { return (qb * TILE + TILE < s ? qb * TILE + TILE : s) - 1; }
// forward: query block qb walks the band key tiles fwd_band_first .. + fwd_band_count - 1, then (if fwd_sees_pivots)
// every pivot tile
__host__ __device__ __forceinline__ int fwd_band_first(int qb, int w, int times) {
    return band_start(qb * TILE, w, times) / TILE;
}
__host__ __device__ __forceinline__ int fwd_band_count(int qb, int s, int w, int times) {
    return last_query(qb, s) / TILE - fwd_band_first(qb, w, times) + 1;
}
__host__ __device__ __forceinline__ bool fwd_sees_pivots(int qb, int s, int w, int times) {
    return band_start(last_query(qb, s), w, times) > 0;
}
// backward band pass: key block kb is visited by query blocks kb .. bwd_band_last
__host__ __device__ __forceinline__ int bwd_band_last(int kb, int nqb, int w, int times) {
    const int e = (((kb * TILE + TILE - 1) / w + times) * w - 1) / TILE;
    return e < nqb - 1 ? e : nqb - 1;
}
// backward pivot pass (launched iff times * w < s): every pivot block is visited by query blocks piv_first .. nqb - 1
// (band_start(i) > 0  <=>  i >= times * w)
__host__ __device__ __forceinline__ int piv_first(int w, int times) { return (times * w) / TILE; }

// Keep bits of the attention-probability dropout: three regions of uint4 (128 bits) entries, each indexed by the
// visiting kernel's own local tile counter so that nothing of size s x s is allocated.
//   fwd  [b, heads, nqb*128 (query), tb + npb, 4]       query-major; slot j = loop index j of the forward
//   band [b, heads, nkb*128 (key),   tq, 4]             key-major;   slot t = query block kb + t of the band pass
//   piv  [b, heads, npb*128 (pivot), np, 4]             key-major;   slot t = query block piv_first + t of the pivot pass
// Word w of a key-major entry holds queries 32w .. 32w + 31 of the block, bit i of word w of a query-major entry key
// 32w + i of the tile.
struct KeepLayout {
    int nqb, nkb, npb;     // query blocks, band key tiles (both ceil(s / 128)), pivot tiles ceil(n_piv / 128)
    int tb, tq, np;        // max band tiles of a forward query block, max query blocks of a band-pass key block,
                           // query blocks of the pivot pass (0 when no query sees a pivot)
    int64_t fwd_words, band_words, piv_words;   // 32-bit words of each region
};

inline KeepLayout keep_layout(int b, int heads, int s, int n_piv, int w, int times) {
    KeepLayout L;
    L.nqb = L.nkb = (s + TILE - 1) / TILE;
    L.npb = (n_piv + TILE - 1) / TILE;
    L.tb = 0;
    L.tq = 0;
    for (int qb = 0; qb < L.nqb; ++qb) {
        const int n = fwd_band_count(qb, s, w, times);
        L.tb = n > L.tb ? n : L.tb;
    }
    for (int kb = 0; kb < L.nkb; ++kb) {
        const int n = bwd_band_last(kb, L.nqb, w, times) - kb + 1;
        L.tq = n > L.tq ? n : L.tq;
    }
    L.np = times * w < s ? L.nqb - piv_first(w, times) : 0;
    const int64_t bh = (int64_t)b * heads;
    L.fwd_words = bh * L.nqb * TILE * (L.tb + L.npb) * 4;
    L.band_words = bh * L.nkb * TILE * L.tq * 4;
    L.piv_words = bh * L.npb * TILE * L.np * 4;
    return L;
}

}  // namespace sparse
}  // namespace cv
