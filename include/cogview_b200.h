/*
 * cogview_b200.h — C ABI of libcogview_b200.so, the sm_90a (H100) implementation of CogView's hot path.
 *
 * The reference (THUDM/CogView) has no FFI: its operator boundary is the Python `mpu` / `model` /
 * `vqvae` namespaces.  Each entry point below replaces the torch/apex/cuBLAS call sequence of one
 * reference function (cited as file:line, relative to the reference tree) and is what a ctypes stub in
 * the reference would bind (INTEGRATION.md shows the stubs).
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless marked host
 *   - functions never allocate or free; the caller owns inputs, outputs and workspaces
 *   - `stream` is a cudaStream_t passed as void*; all work is asynchronous on that stream
 *   - return 0 = ok, < 0 = argument error, > 0 = cudaError_t; cv_last_error() returns the message
 *   - bf16 = __nv_bfloat16 storage; matrices are row-major with a leading dimension in ELEMENTS
 */
#ifndef COGVIEW_B200_H
#define COGVIEW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CV_B200_VERSION 101

int cv_version(void);
const char* cv_last_error(void);
/* number of kernels this library has launched since it was loaded (host-side counter) */
long long cv_launch_count(void);
/* Keep k SMs out of the persistent GEMM grid (returns the SMs it will use): under data parallelism the NCCL kernels of
 * the gradient all-reduce (pretrain_gpt2.py:99-105) run next to the backward GEMMs and need somewhere to live. */
int cv_set_reserved_sms(int k);

/* ------------------------------------------------------------------------------------------------
 * GEMM  C[M,N] = op(A)[M,K] * op(B)[N,K]^T (+ bias[N]) (+ tanh-GELU)      wgmma + TMA
 *   replaces F.linear in ColumnParallelLinear.forward (mpu/layers.py:239-249),
 *   RowParallelLinear.forward (mpu/layers.py:312-326), gelu_impl (mpu/sparse_transformer.py:172-176),
 *   the tied-weight logits GEMM (model/gpt2_modeling.py:117-118) and their autograd backward.
 *   a_mn_major = 0: A stored [M,K] (lda >= K);  1: A stored [K,M] (lda >= M)   (wgrad operand)
 *   b_mn_major = 0: B stored [N,K] (ldb >= K);  1: B stored [K,N] (ldb >= N)   (dgrad/wgrad operand)
 *   C: bf16 (c_is_f32 = 0) or fp32 (c_is_f32 = 1); C2 (optional, bf16, same ld): value before GELU
 *   bias: bf16 [N] or NULL;  act: 0 none, 1 tanh-GELU, 2 ReLU, 3 multiply by gelu'(C2) (C2 = saved pre-activation,
 *         read-only: the GELU backward fused into the dgrad GEMM)
 *   absmax: NULL or device float (must hold a non-negative value): atomic max of |C| — feeds the
 *           reference's abs-max pre-scaled LayerNorm (mpu/sparse_transformer.py:40-44)
 *   block_n: 0 = auto, or 128 / 256
 *   dropout_p > 0: output dropout fused after bias/activation (output_dropout of mpu/sparse_transformer.py:167 and
 *         :233): element (m, n) is kept iff the counter-based generator of site (seed, site) says so, kept values are
 *         scaled by 1/(1-p); abs-max is taken after the dropout.  N % 4 == 0.  dropout_p == 0: no dropout.
 * ---------------------------------------------------------------------------------------------- */
int cv_gemm_bf16(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major, int64_t ldb,
                 void* C, int c_is_f32, int64_t ldc, void* C2, const void* bias, int act, float* absmax,
                 int M, int N, int K, int block_n, float dropout_p, uint64_t seed, uint32_t site, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Abs-max pre-scaled LayerNorm: y = LN(x / (max|x|/8)) * gamma + beta (+ residual)
 *   replaces mpu.LayerNorm.forward (mpu/sparse_transformer.py:40-44) = x.abs().max(), div, apex FusedLayerNorm;
 *   with `residual` it also performs the Sandwich-LN residual add (mpu/sparse_transformer.py:326-329, :337-340).
 *   absmax_in : device float holding max|x| (written by the kernel that produced x, or by cv_absmax)
 *   absmax_out: NULL or device float (>= 0) receiving atomic max |out| (for the next LayerNorm)
 *   mean_out/rstd_out: NULL or [rows] fp32 saved for the backward
 *   supported (x, out, residual): (f32,bf16,-) (bf16,f32,res) (bf16,bf16,-) (f32,f32,-) (f32,f32,res)
 * ---------------------------------------------------------------------------------------------- */
int cv_layernorm_absmax_fwd(const void* x, int x_is_bf16, const float* absmax_in, const void* gamma,
                            const void* beta, float eps, const float* residual, void* out, int out_is_bf16,
                            float* absmax_out, float* mean_out, float* rstd_out, int rows, int cols, void* stream);
int64_t cv_layernorm_bwd_workspace_bytes(int rows, int cols);
/* dx = LN'(dy) (+ dres); dgamma/dbeta bf16 [cols]; workspace of cv_layernorm_bwd_workspace_bytes() bytes.
 * The abs-max scale is a detached constant in the reference (x.abs().max().detach()), and so it is here. */
/* dropout_p > 0: x was the output of dropout site (seed, site) — dx is multiplied by that site's keep mask / (1-p).
 * dxsum (bf16 [cols], may be NULL): column sums of dx — the bias gradient of the linear layer that produced x. */
int cv_layernorm_absmax_bwd(const void* x, int x_is_bf16, const void* dy, int dy_is_bf16, const float* mean,
                            const float* rstd, const void* gamma, const float* dres, void* dx, int dx_is_bf16,
                            void* dgamma, void* dbeta, float* workspace, int rows, int cols, float dropout_p,
                            uint64_t seed, uint32_t site, void* dxsum, void* stream);
int cv_absmax(const void* x, int x_is_bf16, int64_t n, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense attention forward: ctx = softmax((Q/sqrt(hn)) K^T * mask - 10000 (1 - mask)) V
 *   replaces standard_attention (mpu/sparse_transformer.py:652-673) and the split/permute/contiguous copies
 *   of GPT2ParallelSelfAttention.forward (mpu/sparse_transformer.py:131-163).
 *   q: [b, sq, heads*64], k/v: [b, sk, heads*64] bf16 with row stride ld* and batch stride bs* (elements) —
 *   e.g. three views into the packed QKV GEMM output.  Queries are the LAST sq of the sk positions.
 *   mask: key j visible to query i iff j < sep + (sk - sq) or j <= i + (sk - sq)
 *         (sep = 0: lower-triangular mask of pretrain_gpt2.py:218-221; sep > 0: the int-`sep` form of
 *          mpu/sparse_transformer.py:477-489)
 *   out: [b, sq, heads*64] bf16 (token-major, what the out-projection GEMM reads); lse: NULL or [b, heads, sq]
 *   dropout_p > 0: dropout on the attention probabilities (torch.nn.Dropout under the RNG-tracker fork,
 *         mpu/sparse_transformer.py:667-669).  The keep decisions are generated by a separate full-occupancy kernel
 *         launched by this call: one Philox4x32-10 call per (query, 128-key tile) of the counter-based generator
 *         (seed, site) seeds four 32-step LCG streams, keep iff state >= p * 2^32.
 *         drop_mask: uint32 buffer of 2 * b * heads * ceil(sk/128) * ceil(sq/128) * 128 * 4 words, two regions:
 *           [0] key-major   [b, heads, ceil(sk/128)*128, ceil(sq/128), 4]: bit i of word w of (key, query block qb)
 *               is query qb*128 + 32w + i — what cv_attn_bwd reads (pass the same pointer);
 *           [1] query-major [b, heads, ceil(sq/128)*128, ceil(sk/128), 4]: consumed by the forward kernel.
 *         Tiles that the mask never makes visible are left unwritten.
 * ---------------------------------------------------------------------------------------------- */
int cv_attn_fwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk, const void* v,
                int64_t ldv, int64_t bsv, void* out, int64_t ldo, int64_t bso, float* lse, int b, int heads,
                int head_dim, int sq, int sk, int sep, float dropout_p, uint64_t seed, uint32_t site,
                uint32_t* drop_mask, void* stream);

/* Backward of cv_attn_fwd for sq == sk (training).  q/k/v as in cv_attn_fwd; out, d_out: [b, s, heads*64] bf16
 * contiguous; lse from the forward; dropout_p > 0: drop_mask is the buffer the forward filled (region [0] is read).  dqkv: [b, s, 3*heads*64] bf16 (dQ | dK | dV, the layout of the packed QKV
 * GEMM output, so the QKV dgrad/wgrad GEMMs read it directly).  workspace: cv_attn_bwd_workspace_bytes(). */
int64_t cv_attn_bwd_workspace_bytes(int b, int heads, int head_dim, int s);
int cv_attn_bwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk, const void* v,
                int64_t ldv, int64_t bsv, const void* out, const void* d_out, const float* lse, void* dqkv,
                void* workspace, int b, int heads, int head_dim, int s, int sep, float dropout_p,
                const uint32_t* drop_mask, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Embedding: hidden = wte[ids] + wpe[pos] (fp32) and max|hidden|
 *   replaces VocabParallelEmbedding.forward (mpu/layers.py:117-133) + position add (mpu/sparse_transformer.py:522-523)
 * ---------------------------------------------------------------------------------------------- */
int cv_embed_fwd(const int64_t* ids, const int64_t* pos, const void* wte, const void* wpe, float* out,
                 float* absmax, int rows, int hidden, float dropout_p, uint64_t seed, uint32_t site, void* stream);
int cv_embed_bwd(const int64_t* ids, const int64_t* pos, const float* dx, void* dwte, void* dwpe, int rows,
                 int hidden, float dropout_p, uint64_t seed, uint32_t site, void* stream);
/* keep mask (1 = kept) of the first n elements of dropout site (seed, site) — the pure function of
 * (seed, site, element index) that every fused dropout in this library uses; exposed for tests. */
int cv_dropout_mask(uint8_t* out, int64_t n, float p, uint64_t seed, uint32_t site, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Vocab cross-entropy on fp32 logits — mpu/cross_entropy.py:27-104 at model-parallel size 1.
 *   fwd: loss[r], and the row max / sum(exp) saved for bwd;  bwd: dlogits (bf16) = (softmax - onehot) * grad_loss[r]
 * ---------------------------------------------------------------------------------------------- */
int cv_cross_entropy_fwd(const float* logits, int64_t ld, const int64_t* target, float* loss, float* row_max,
                         float* row_sum, int rows, int vocab, void* stream);
int cv_cross_entropy_bwd(const float* logits, int64_t ld, const int64_t* target, const float* row_max,
                         const float* row_sum, const float* grad_loss, void* dlogits, int64_t ldd, int rows,
                         int vocab, void* stream);

/* GELU backward (mpu/sparse_transformer.py:172-176): dpre = dact * gelu'(pre), bf16, n % 8 == 0 */
/* dst[i] += src[i] for i < n, fp32; n a multiple of 4, both 16-byte aligned. */
int cv_add_f32(float* dst, const float* src, int64_t n, void* stream);

int cv_gelu_bwd(const void* pre, const void* dact, void* dpre, int64_t n, void* stream);
/* bias gradient: out[c] = sum_r dy[r, c] (bf16 in/out, fp32 accumulate) */
int64_t cv_colsum_workspace_bytes(int cols);
int cv_colsum_bf16(const void* dy, int64_t ld, void* out, float* workspace, int rows, int cols, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sparse TRAINING attention: sparse_attention + _chunk (mpu/sparse_transformer.py:675-725, :629-650) with the
 * pivot mask of :491-496 / :569 in closed form.  One softmax over
 *     band   : keys j with band_start(i) <= j <= i,  band_start(i) = max(0, i / w - times + 1) * w
 *     pivots : the n_piv gathered keys K[pivot_idx], V[pivot_idx] whose position is < band_start(i), scores + log(s / n_piv)
 * walked by ONE flash kernel as band tiles followed by gathered-pivot tiles (wgmma + TMA, same kernel as cv_attn_fwd);
 * masked entries carry exactly -10000 as in the reference.  q / k / v: [b, s, heads*64] bf16 views as for cv_attn_fwd;
 * pivot_idx: int64 [b, n_piv] (distinct positions per sequence, mpu/sparse_transformer.py:557-565); s % w == 0.
 * The backward runs the band pass and the pivot pass with the joint lse / delta, scatters the pivot dK / dV back and
 * writes dqkv [b, s, 3*heads*64] (dQ | dK | dV).
 * ---------------------------------------------------------------------------------------------- */
int64_t cv_attn_sparse_workspace_bytes(int b, int heads, int head_dim, int n_piv);
int cv_attn_sparse_fwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk, const void* v,
                       int64_t ldv, int64_t bsv, const int64_t* pivot_idx, void* out, int64_t ldo, int64_t bso,
                       float* lse, void* workspace, int b, int heads, int head_dim, int s, int n_piv, int query_window,
                       int key_window_times, float dropout_p, uint64_t seed, uint32_t site, uint32_t* drop_mask,
                       void* stream);
int64_t cv_attn_sparse_bwd_workspace_bytes(int b, int heads, int head_dim, int s, int n_piv);
int cv_attn_sparse_bwd(const void* q, int64_t ldq, int64_t bsq, const void* k, int64_t ldk, int64_t bsk, const void* v,
                       int64_t ldv, int64_t bsv, const int64_t* pivot_idx, const void* out, const void* d_out,
                       const float* lse, void* dqkv, void* workspace, int b, int heads, int head_dim, int s, int n_piv,
                       int query_window, int key_window_times, float dropout_p, const uint32_t* drop_mask,
                       void* stream);
/* dropout_p > 0: dropout on the joint pivot + band probabilities (attention_dropout of mpu/sparse_transformer.py:719-721):
 * the row sum and lse stay undropped, the 1/(1-p) scale is applied once to the output row, and the backward sends dP and
 * dV through the keep bits.  The keep decision of (query i, key) is a pure function of (seed, site, batch, head, i,
 * virtual key), where the virtual keys are the s sequence positions (band keys) followed by the n_piv pivot SLOTS: pivot
 * p is decided as column p of the reference's [b, heads, s, n_piv + w*times] probabilities, whatever its position.
 * One Philox4x32-10 call of counter ((batch*heads + head)*s + i) * (nkb + npb) + virtual key tile seeds four 32-step
 * LCG streams (key 32g + t of the tile is step t of stream g), keep iff state >= p * 2^32.
 *   drop_mask: uint32 buffer of cv_attn_sparse_drop_mask_words() words, filled by the forward and read by the backward
 *   (pass the same pointer), three regions in this order, with nqb = nkb = ceil(s/128), npb = ceil(n_piv/128):
 *     [fwd]  query-major [b, heads, nqb*128 (query), TB + npb, 4]: bit t of word g of (query i, slot j) is key 32g + t of
 *            the j-th tile query block i/128 visits: band key tiles jb0 .. jb0 + nband - 1 (jb0 = band_start(128 qb)/128,
 *            nband = last query of the block / 128 - jb0 + 1), then, if band_start(last query) > 0, pivot tiles 0 .. npb-1
 *            at slots nband .. nband + npb - 1.  TB = the largest nband.
 *     [band] key-major [b, heads, nkb*128 (key), TQ, 4]: bit t of word g of (key, slot u) is query 128 (kb + u) + 32g + t,
 *            kb = key / 128, for u = 0 .. i_end(kb) - kb, i_end(kb) = min(nqb - 1, ((((kb+1)*128 - 1) / w + times) * w - 1) / 128).
 *            TQ = the largest i_end(kb) - kb + 1.
 *     [piv]  key-major [b, heads, npb*128 (pivot slot), NP, 4]: bit t of word g of (pivot p, slot u) is query
 *            128 (i0 + u) + 32g + t, i0 = (times*w) / 128; NP = nqb - i0 when times*w < s, else 0 (no query sees a pivot).
 *   Entries that neither kernel reads are left unwritten.
 * dropout_p == 0: no dropout; drop_mask may be NULL. */
int64_t cv_attn_sparse_drop_mask_words(int b, int heads, int s, int n_piv, int query_window, int key_window_times);

/* ------------------------------------------------------------------------------------------------
 * Decode (one new token per sequence): HBM-bound weight streaming, CUDA cores.
 *   cv_linear_small_m: y[M,N] = x[M,K] W[N,K]^T + bias (+GELU) (+abs-max), 1 <= M <= 16 — F.linear of
 *     mpu/layers.py:243,319 and the last-token logits GEMM (model/gpt2_modeling.py:117) inside the sampling
 *     loop (generation/sampling.py:147-155).  out bf16 or fp32.
 *   cv_attn_decode: standard_attention (mpu/sparse_transformer.py:652-673) for sq = 1 over a K|V cache
 *     [b, max_len, 2*heads*64]; qkv [b, 3*heads*64] holds q | k_new | v_new of the token at position cur_len,
 *     which is appended to the cache by the same kernel.  cur_len comes from *cur_len_dev when non-NULL
 *     (so a captured CUDA graph can be replayed), else from cur_len.  out [b, heads*64] bf16.  row_pad (device int32
 *     [b] or NULL) gives a cache length per sequence, for a batch whose rows come from prompts of different lengths:
 *     row b holds t_b = cur_len - row_pad[b] cached tokens (cur_len: the longest row), attends over its keys 0..t_b,
 *     the new token last, and appends its K|V at slot t_b; slots above t_b are neither read nor written.  Contract:
 *     0 <= row_pad[b] <= cur_len and t_b < max_len.  With row_pad all zero, out and cache are bit-identical to
 *     row_pad == NULL at the same nsplit.
 * ---------------------------------------------------------------------------------------------- */
int cv_linear_small_m(const void* x, int64_t ldx, const void* W, int64_t ldw, const void* bias, void* out,
                      int64_t ldo, int out_is_f32, int act, float* absmax, int M, int N, int K, void* stream);
/* Sandwich-LN glue between two decode linears (M <= 16, one CTA): y = res_in + LN_post(gemm_out) (skipped when
 * gemm_out is NULL), xn = LN_pre(y) with both abs-max pre-scales (mpu/sparse_transformer.py:40-44, :319-331, :337-340).
 * res_out (fp32, may be NULL) receives y; xn_out (bf16) feeds the next linear. */
int cv_ln_pair_small_m(const float* res_in, const void* gemm_out, const float* absmax_gemm, const void* g_post,
                       const void* b_post, const void* g_pre, const void* b_pre, float eps, float* res_out,
                       void* xn_out, int M, int K, void* stream);
/* The same two operations for 17 <= M <= 64 rows (csrc/decode_mid.cu), same arguments.
 *   cv_linear_mid_m: TMA + wgmma weight streaming with the weights as the 64-row operand; K is split over the CTAs
 *     of a thread-block cluster and reduced in a fixed order through distributed shared memory, so equal inputs give
 *     equal bits.  W is read through a tensor map: ldw * 2 bytes must be a multiple of 16 (ldw % 8 == 0).
 *   cv_ln_pair_mid_m: one cluster of ceil(M / 8) CTAs; max|y| over all rows is exchanged through distributed shared
 *     memory.  K <= 2560. */
int cv_linear_mid_m(const void* x, int64_t ldx, const void* W, int64_t ldw, const void* bias, void* out, int64_t ldo,
                    int out_is_f32, int act, float* absmax, int M, int N, int K, void* stream);
int cv_ln_pair_mid_m(const float* res_in, const void* gemm_out, const float* absmax_gemm, const void* g_post,
                     const void* b_post, const void* g_pre, const void* b_pre, float eps, float* res_out, void* xn_out,
                     int M, int K, void* stream);
/* sparse_attention_inference (mpu/sparse_transformer.py:727-750): dense softmax over the gathered keys
 * K[idx], V[idx] (idx = pivots U trailing window, [b, n] int64; its last sq entries are the queries' own positions,
 * which get the causal -10000 above the diagonal).  q: [b, sq, heads*64] view; cache [b, max_len, 2*heads*64] (K|V)
 * already holding the new tokens; out [b, sq, heads*64] bf16 contiguous. */
int cv_attn_gather(const void* q, int64_t ldq, int64_t bsq, const void* cache, int64_t cache_batch_stride,
                   const int64_t* idx, void* out, int b, int heads, int head_dim, int sq, int n, void* stream);
int64_t cv_attn_decode_workspace_bytes(int b, int heads, int nsplit);
int cv_attn_decode(const void* qkv, void* cache, int64_t cache_batch_stride, const int* cur_len_dev, int cur_len,
                   const int* row_pad, void* out, float* workspace, int b, int heads, int head_dim, int max_len,
                   int nsplit, void* stream);
/* Ragged multi-token attention on the K|V cache (csrc/attn_chunk.cu): a chunk of n new tokens per sequence.
 * qkv [b, n, 3h] bf16 is the packed QKV GEMM output (q | k | v per token, token-major, read in place); cache
 * [b, max_len, 2h] bf16 (K | V) with batch stride cache_batch_stride elements; row_pad device int32 [b] or NULL.
 * Row r holds t_r = cur_len - row_pad[r] cached tokens (t_r = cur_len for every row when row_pad is NULL).  Query i of
 * row r (position t_r + i) attends keys 0 .. t_r + i: the row's cache, then the chunk causally; no sep.  Softmax of
 * the scores scaled by 1/sqrt(64), as standard_attention.  The chunk's K|V is written at slots t_r .. t_r + n - 1 and
 * nothing else in the cache is written.  out [b, n, h] bf16 (token-major, the out-projection GEMM's input).
 * nsplit > 1 splits every row's keys over that many CTAs and merges them in a second kernel; it needs workspace of
 * cv_attn_chunk_workspace_bytes(b, heads, n, nsplit) bytes.  Argument errors: head_dim != 64, n outside 1..64,
 * cur_len + n > max_len, nsplit outside 1..64, misaligned pointers.  Contract (not checked, device data):
 * 0 <= row_pad[r] <= cur_len. */
int64_t cv_attn_chunk_workspace_bytes(int b, int heads, int n, int nsplit);
int cv_attn_chunk_ragged(const void* qkv, void* cache, int64_t cache_batch_stride, int cur_len, const int* row_pad,
                         void* out, float* workspace, int b, int n, int heads, int head_dim, int max_len, int nsplit,
                         void* stream);
/* standard_attention (mpu/sparse_transformer.py:652-673) for sq = 1, as cv_attn_decode, for rows that share a prompt
 * (csrc/attn_shared.cu): the beams of one image in image-to-text sampling (generate_samples.py:161-186).  The b rows
 * form `groups` groups of G = b / groups consecutive rows; the prompt's K|V is held once per group.
 * qkv [b, 3h] bf16: q | k_new | v_new of each row.  prefix [groups, max_len, 2h] bf16 (K | V, batch stride
 * prefix_batch_stride elements), read only: every group's prompt is prefix_len = P tokens long.  suffix [b, s_max, 2h]
 * bf16 (K | V, batch stride suffix_batch_stride): row r's generated tokens.  The suffix length s comes from *s_dev when
 * non-NULL (so a captured CUDA graph can be replayed), else from s.  Row r of group g = r / G attends, in this order,
 * to prefix[g, 0:P], suffix[r, 0:s] and its new key: softmax of the scores scaled by 1/sqrt(64).  Row r's k|v is
 * written at suffix[r, s]; nothing else in either buffer is written.  out [b, h] bf16.  Every prefix key and value is
 * read once per (group, head); nsplit (1..64) splits the prefix keys over that many CTAs, and a second kernel per
 * (row, head) adds the suffix and the new key and merges.  workspace: cv_attn_shared_workspace_bytes(b, heads, nsplit)
 * bytes, always required.  Argument errors: head_dim != 64, G outside 1..64 or b % groups != 0, P > max_len,
 * s >= s_max (s from the host), nsplit outside 1..64, misaligned pointers.  Contract (not checked, device data):
 * 0 <= *s_dev < s_max. */
int64_t cv_attn_shared_workspace_bytes(int b, int heads, int nsplit);
int cv_attn_decode_shared(const void* qkv, const void* prefix, int64_t prefix_batch_stride, int prefix_len, int max_len,
                          void* suffix, int64_t suffix_batch_stride, const int* s_dev, int s, int s_max, void* out,
                          float* workspace, int b, int groups, int heads, int head_dim, int nsplit, void* stream);
/* Sparse inference (is_sparse == 2, mpu/sparse_transformer.py:498-520, :591-600, :727-750) without the host:
 *   cv_sparse_plan: the key index list of one decode step for EVERY layer: idx [num_layers, b, nmax] int32, *n_dev = its
 *     length.  Per (layer, sequence): every text position before the trailing window (is_txt [b, max_len] uint8 marks
 *     them), a uniformly random subset of the image positions before it — num_pivot_now = max_text +
 *     int((left_boundary - max_text) * num_pivot / max_sequence_length) entries in total, as :508-510 — then the window
 *     [left_boundary, *cur_len_dev].  The subset is drawn with counter-based random keys (seed *seed_dev, the step, the
 *     layer, the sequence, the position): the distribution of random.sample, not its stream.  *err is set to 1 if the
 *     list does not fit nmax.  batch <= 16, positions <= 4096.
 *   cv_attn_decode_gather: cv_attn_decode over that key list (idx + batch * idx_batch_stride, *n_dev entries; the new
 *     token's position *cur_len_dev must be in the list — it is the last window entry) with the same fused append. */
int cv_sparse_plan(const void* is_txt, int64_t txt_batch_stride, const int* cur_len_dev, int num_layers, int b, int window,
                   int num_pivot, int max_sequence_length, const void* seed_dev, int* idx, int nmax, int* n_dev, int* err,
                   void* stream);
int cv_attn_decode_gather(const void* qkv, void* cache, int64_t cache_batch_stride, const int* cur_len_dev, const int* idx,
                          int64_t idx_batch_stride, const int* n_dev, void* out, float* workspace, int b, int heads,
                          int head_dim, int max_len, int nsplit, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sampling epilogue of the decode loop in one kernel (one CTA per sequence): generation/sampling.py:157-183 with
 * top_k_logits (:24-33) — logits / temperature, invalid vocabulary slices, keep every logit >= the k-th largest
 * (exact radix select; ties at the threshold are all kept, as `logits < kth` does), softmax over the kept ones,
 * one multinomial draw (counter-based Philox: seed, draw index = *step, sequence), log-probability of the draw.
 *   seed: *seed_dev when seed_dev != NULL (so that a captured graph can be re-seeded), else `seed`.
 *   logits fp32 [b, ld] (not modified); valid: HOST array of n_valid (<= 4) [lo, hi) vocabulary ranges = the
 *   complement of the reference's invalid_slices; top_k <= 0 keeps everything valid.
 *   Outputs (all device, any may be NULL except next_ids): next_ids int64 [b] <- the draw; out_tokens int64
 *   [b, ld_out] column *step <- the draw; score_acc fp32 [b] += log p(draw); pos int64 [b] += 1; cur_len int32 += 1;
 *   step int64 += 1 (the shared scalars are advanced by the last CTA to finish); probs_out fp32 [b, ld] (testing):
 *   the full post-filter distribution.
 *   top_p > 0: nucleus (top-p) filtering after the top-k filter (top_k_logits :34-47): of the top-k survivors, keep a
 *   token iff the probability mass of the tokens strictly above it (softmax over the survivors) is <= top_p; the first
 *   token that takes the mass past top_p is kept.  Every token whose logit equals the boundary logit is kept
 *   (torch.sort leaves the order among ties unspecified).  The mass is accumulated in 2^-40 fixed point (exact integer
 *   sums: repeated calls are bit-equal).  top_p >= 1 keeps every top-k survivor; top_p <= 0: no nucleus filter.
 * ---------------------------------------------------------------------------------------------- */
int cv_sample_topk(const float* logits, int64_t ld, int b, int vocab, float temperature, int top_k,
                   const int* valid, int n_valid, uint64_t seed, const uint64_t* seed_dev, int64_t* step,
                   int64_t* next_ids, int64_t* out_tokens, int64_t ld_out, float* score_acc, int64_t* pos, int* cur_len,
                   unsigned int* done_counter, float* probs_out, float top_p, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Optimizer step: fused AdamW on bf16 parameters with fp32 master weights / moments — replaces
 * FP16_Optimizer.step + apex FusedAdam (fp16/fp16.py:399-453, pretrain_gpt2.py:139-140; decoupled weight decay)
 * and, with cv_sumsq_bf16_multi + cv_clip_coef, the global-norm clipping of mpu/grads.py:28-74.
 * One launch over a device-resident table (the whole parameter list of a model).
 *   grad_scale_dev: NULL or device float multiplied into the gradient (the clip coefficient).
 *   param / grad 8-byte aligned, master / m / v 16-byte aligned (for cv_sumsq_bf16_multi, grad 16-byte aligned);
 *   bias_correction{1,2} = 1 - beta{1,2}^step, step >= 1.
 * ---------------------------------------------------------------------------------------------- */
typedef struct cv_adamw_entry {
    void* param;          /* bf16 [n] */
    const void* grad;     /* bf16 [n] */
    float* master;        /* fp32 [n] */
    float* m;             /* fp32 [n] */
    float* v;             /* fp32 [n] */
    int64_t n;
    float lr, weight_decay, bias_correction1, bias_correction2;
} cv_adamw_entry;         /* 64 bytes */
/* state (device int[2], may be NULL): [0] = 1 when this step is skipped, [1] = number of applied steps.
 * cv_clip_coef sets state[0] = 1 (and coef = 0) when the gradient norm is inf/NaN — the overflow branch of
 * FP16_Optimizer.step (fp16/fp16.py:399-420) — else state[0] = 0 and state[1] += 1; cv_adamw_step_multi with a
 * non-NULL state leaves everything untouched on a skipped step and takes the bias corrections from state[1]
 * instead of the table. */
int cv_adamw_step_multi(const cv_adamw_entry* table_dev, int count, float beta1, float beta2, float eps,
                        const float* grad_scale_dev, float grad_scale, const int* state, void* stream);
/* *out += sum(grad^2) over .grad / .n of every entry */
int cv_sumsq_bf16_multi(const cv_adamw_entry* table_dev, int count, float* out, void* stream);
int cv_clip_coef(const float* sumsq, float max_norm, float* coef, float* norm_out, int* state, void* stream);

/* ------------------------------------------------------------------------------------------------
 * VQ-VAE image tokenizer (vqvae/vqvae_zc.py, vqvae/api.py), NHWC bf16 activations.
 *   cv_conv2d_k4s2 / cv_conv_transpose2d_k4s2: nn.Conv2d / nn.ConvTranspose2d (kernel 4, stride 2, padding 1) of
 *     Encoder (vqvae_zc.py:121-129) and Decoder (:172-191) as im2col-free implicit GEMMs on wgmma: A tiles are
 *     TMA boxes of the NHWC input (traversal stride 2 / sub-pixel phases, zero-filled halo = padding).
 *     x: [B, IH, IW, Cin]; w_packed: [16 (ky*4+kx), Cout, Cin] bf16; bias bf16 [Cout] or NULL; relu fused.
 *     y: [B, IH/2, IW/2, Cout] (conv) or [B, 2IH, 2IW, Cout] (transposed).  Cin % 64 == 0, Cout % 128 == 0.
 *     Tile grid (output for the conv, input for the transposed conv) [B, H, W]: either H, W powers of two with
 *     W <= 128 (128-pixel tiles of whole rows or whole images; B must be a multiple of 128 / (H W) when H W < 128),
 *     or W > 128 with W % 128 == 0 and any H >= 1 (128-pixel row segments).  Other shapes are refused.
 *   cv_im2col_k4s2_c3: patches of the fp32 NCHW 3-channel image -> [B*OH*OW, 64] bf16 (48 used) for the first conv
 *     (run as cv_gemm_bf16 with act = 2).
 *   cv_vq_split3 / cv_vq_argmin / cv_vq_lookup: Quantize.forward_ hard path (vqvae_zc.py:41-54) and embed_code (:95-96);
 *     scores = split3(z) . [E_hi|E_lo|E_hi]^T via cv_gemm_bf16 (fp32 out); argmin of e2[j] - 2 scores[j] with exact
 *     fp32 re-scoring of the two best codes when closer than `margin` (relative); ties -> lowest index.
 *   cv_conv1x1_out3: Decoder's final 1x1 conv to 3 channels (:191) + de-normalisation of vqvae/api.py:43, NCHW fp32 out.
 * ---------------------------------------------------------------------------------------------- */
int cv_conv2d_k4s2(const void* x, const void* w_packed, const void* bias, void* y, int B, int IH, int IW, int Cin,
                   int Cout, int relu, void* stream);
int cv_conv_transpose2d_k4s2(const void* x, const void* w_packed, const void* bias, void* y, int B, int IH, int IW,
                             int Cin, int Cout, int relu, void* stream);
int cv_im2col_k4s2_c3(const float* img, void* out, int B, int H, int W, void* stream);
int cv_vq_split3(const float* z, void* out, int64_t rows, int dim, void* stream);
int cv_vq_argmin(const float* scores, int64_t ld, const float* e2, const float* z, const float* codebook,
                 int64_t* idx_out, int64_t rows, int n_embed, int dim, float margin, void* stream);
int cv_vq_lookup(const int64_t* idx, const float* codebook, void* out_bf16, float* out_f32, int64_t rows, int dim,
                 void* stream);
int cv_conv1x1_out3(const void* x, const float* w, const float* bias, const float* scale, const float* shift,
                    float* out, int B, int H, int W, int cin, void* stream);

/* ------------------------------------------------------------------------------------------------
 * VQ-VAE training (vqvae_zc.py in train() mode).  Every reduction runs in a fixed order: equal inputs, equal bits.
 *   cv_conv_k4s2_wgrad: weight gradient of a k4 s2 p1 Conv2d or ConvTranspose2d.  With the small map
 *     S [B, h, w, M] and the big map G [B, 2h, 2w, N] (NHWC bf16),
 *       out[m, n, ky, kx] = sum_{b,y,x} S[b, y, x, m] * G[b, 2y - 1 + ky, 2x - 1 + kx, n]   (zero outside G), fp32.
 *     Conv2d: S = dY, G = X -> dW [Cout, Cin, 4, 4].  ConvTranspose2d: S = X, G = dY -> dW [Cin, Cout, 4, 4].
 *     M % 128 == 0, N % 256 == 0; workspace of cv_conv_k4s2_wgrad_workspace_bytes (split-K partials).
 *   cv_relu_mask_bf16: dx[i] = act[i] > 0 ? dx[i] : 0 in place (act = the saved ReLU output); n % 8 == 0.
 *   cv_conv1x1_out3_bwd: backward of the Decoder's last 1x1 conv (:191) from dr = dL/d(out) [B, 3, H, W] fp32 and
 *     the saved ReLU output x [B, H, W, cin] bf16: dx = (dr . w) * (x > 0) bf16 NHWC, dw [3, cin] and db [3] fp32.
 *     cin = 8 x a divisor of 256; workspace of cv_conv1x1_out3_bwd_workspace_bytes.
 *   cv_vq_ema_stats: embed_onehot_sum (counts [n_embed]) and embed_sum = flatten^T . onehot ([dim, n_embed]) of
 *     Quantize.forward_ (:68-69) from the codes idx [rows] and z [rows, dim] fp32; each code's rows are summed in
 *     row order.
 * ---------------------------------------------------------------------------------------------- */
int64_t cv_conv_k4s2_wgrad_workspace_bytes(int B, int h, int w, int M, int N);
int cv_conv_k4s2_wgrad(const void* S, const void* G, float* out, float* workspace, int B, int h, int w, int M, int N,
                       void* stream);
int cv_relu_mask_bf16(void* dx, const void* act, int64_t n, void* stream);
int64_t cv_conv1x1_out3_bwd_workspace_bytes(int cin);
int cv_conv1x1_out3_bwd(const float* dr, const void* x, const float* w, void* dx, float* dw, float* db,
                        float* workspace, int B, int H, int W, int cin, void* stream);
int cv_vq_ema_stats(const int64_t* idx, const float* z, int64_t rows, int dim, int n_embed, float* counts,
                    float* embed_sum, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Gumbel-softmax quantiser (vqvae_zc.py, Quantize.forward_ with continuous_relax=True: soft :55-60, hard :61-65,
 * the KL :89-90, gumbel_softmax :284-346).  Row r of the fp32 scores s [rows, ld] is z_r . E (the split3 GEMM of the
 * nearest-code path) and e2 [K] is |e_j|^2, so a_rj = 2 s_rj - e2_j is -dist up to the row constant |z_r|^2, which
 * cancels in every softmax and arg-max.  K % 4 == 0; row indices row0 + r < 2^32.  One CTA per row, every reduction
 * in a fixed order: equal inputs give equal bits.
 *   cv_gumbel_noise: the noise g[r, j] = -log(-log(u)) of absolute row row0 + r and code j, u in [2^-24, 1 - 2^-24]
 *     from Philox4x32-10 under `seed`; a function of (seed, absolute row, code) alone.  out: [rows, K] fp32.
 *   cv_vq_gumbel_fwd: y = softmax((a + g) / tau) (:333-334), written as bf16 (y_f32 = 0) or fp32 (y_f32 = 1) rows of
 *     stride ldy, or not at all (y = NULL: the hard relaxation needs only the index); idx = the arg-max of (a + g) / tau,
 *     the lowest index on ties (:338, :345); kl[r] = sum_j qy_j log(qy_j K + 1e-20) with qy = softmax(a) (:89-90),
 *     or NULL.
 *   cv_vq_gumbel_bwd: from dy = dL/dy [rows, lddy] fp32 (NULL: no y term) and kl_scale = dL/d(KL mean) / total rows
 *     (0: no KL term), da = y (dy - <y, dy>) / tau + kl_scale qy (h - <qy, h>) with
 *     h_j = log(qy_j K + 1e-20) + qy_j K / (qy_j K + 1e-20), written as bf16 [rows, ldda]; rowsum[r] = sum_j da_rj
 *     (fp32, before rounding), for the -2 z rowsum(da) term of d(-dist)/dz.  y and qy are regenerated from s and the
 *     noise, so nothing but z needs to be kept between the forward and the backward.
 * ---------------------------------------------------------------------------------------------- */
int cv_gumbel_noise(uint64_t seed, int64_t row0, int64_t rows, int K, float* out, void* stream);
int cv_vq_gumbel_fwd(const float* s, int64_t ld, const float* e2, int64_t rows, int K, uint64_t seed, int64_t row0,
                     float tau, void* y, int y_f32, int64_t ldy, int64_t* idx, float* kl, void* stream);
int cv_vq_gumbel_bwd(const float* s, int64_t ld, const float* e2, int64_t rows, int K, uint64_t seed, int64_t row0,
                     float tau, const float* dy, int64_t lddy, float kl_scale, void* da, int64_t ldda, float* rowsum,
                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * Token log-probabilities over a vocabulary window, without logits in global memory (post-selection: the caption
 * log-likelihood of generation/sampling.py:214-230, log(softmax) of the logits with the image vocabulary at -inf).
 *   logp[m] = H[m] . W[target[m]] - logsumexp_{v_begin <= v < v_end} H[m] . W[v]; -inf when target[m] lies outside
 *   [v_begin, v_end).  H bf16 [M, K] (ldh), W bf16 [V >= v_end, K] (ldw; the tied word embedding), target int64 [M],
 *   logp fp32 [M].  K, ldh and ldw follow cv_gemm_bf16 (multiples of 8); M >= 1 and the window width are arbitrary.
 *   A wgmma GEMM whose epilogue keeps one (max, sum exp) pair per (row, 256-column tile), then one reduction per row
 *   in column-tile order: equal inputs give equal bits.  workspace: cv_vocab_logprob_workspace_bytes(M, v_begin,
 *   v_end) bytes, 8-byte aligned, need not be initialised.
 * ---------------------------------------------------------------------------------------------- */
int64_t cv_vocab_logprob_workspace_bytes(int M, int v_begin, int v_end);
int cv_vocab_logprob(const void* H, int64_t ldh, const void* W, int64_t ldw, const int64_t* target, float* logp,
                     float* workspace, int M, int K, int v_begin, int v_end, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Vocabulary cross-entropy for training without logits in global memory: the per-token loss of
 * mpu/cross_entropy.py:27-104 over the whole vocabulary [0, V), with its gradient recomputed per column window.
 *   H bf16 [M, K] (ldh), W bf16 [V, K] (ldw; the tied word embedding), target int64 [M]; K, ldh and ldw follow
 *   cv_gemm_bf16 (multiples of 8, H and W 16-byte aligned); M >= 1 and V are arbitrary.
 * cv_vocab_xent_fwd: loss[m] = lse[m] - H[m] . W[target[m]], lse[m] = logsumexp_{0 <= v < V} H[m] . W[v], both fp32
 *   [M], from the fp32 accumulators of a wgmma GEMM (the logits route rounds the same values; only the order of the
 *   sum of exponentials differs).  A target outside [0, V) gives loss NaN (lse is still written).  workspace:
 *   cv_vocab_xent_workspace_bytes(M, V) bytes, 8-byte aligned, need not be initialised.  The row's partial
 *   (max, sum exp) pairs are folded in column-tile order: equal inputs give equal bits.
 * cv_vocab_xent_dlogits: for the window [v_begin, v_end) (0 <= v_begin < v_end <= V)
 *   D[m, v - v_begin] = bf16(grad_loss[m] * (exp(H[m] . W[v] - lse[m]) - [v == target[m]])),
 *   lse from cv_vocab_xent_fwd, grad_loss fp32 [M].  D bf16 [M, ldd], ldd >= v_end - v_begin and even, D 4-byte
 *   aligned; columns at or past v_end - v_begin and rows past M are not written.  A target outside the window
 *   subtracts nothing there.  Each element is computed once from a fixed-order GEMM, with no atomics: equal inputs
 *   give equal bits.
 * ---------------------------------------------------------------------------------------------- */
int64_t cv_vocab_xent_workspace_bytes(int M, int V);
int cv_vocab_xent_fwd(const void* H, int64_t ldh, const void* W, int64_t ldw, const int64_t* target, float* loss,
                      float* lse, float* workspace, int M, int K, int V, void* stream);
int cv_vocab_xent_dlogits(const void* H, int64_t ldh, const void* W, int64_t ldw, const int64_t* target,
                          const float* lse, const float* grad_loss, void* D, int64_t ldd, int M, int K, int v_begin,
                          int v_end, void* stream);

#ifdef __cplusplus
}
#endif
#endif
