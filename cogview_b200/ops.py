"""Thin functional wrappers over the C ABI: allocate outputs with torch, pass raw pointers + stream.

These are the only places that call into libcogview_b200.so; the `mpu` / `model` / `vqvae` mirrors of the
reference interface are built on them.
"""
import torch

from . import _lib
from ._lib import check, lib, ptr, require_cuda, stream_ptr

ACT_NONE = 0
ACT_GELU = 1
ACT_RELU = 2
ACT_GELU_GRAD = 3   # multiply the result by gelu'(aux) (GELU backward fused into the dgrad GEMM)


def gemm(a, b, *, a_mn_major=False, b_mn_major=False, bias=None, act=ACT_NONE, out_dtype=torch.bfloat16,
         absmax=None, want_preact=False, out=None, block_n=0, aux=None, dropout=None):
    """C[M,N] = op(A)[M,K] @ op(B)[N,K]^T (+bias) (+GELU).

    a: [M,K] (or [K,M] when a_mn_major); b: [N,K] (or [K,N] when b_mn_major); both bf16, last dim contiguous.
    absmax: optional 1-element fp32 tensor updated with atomic max |C|.
    Returns C, or (C, preact) when want_preact.
    """
    require_cuda(a, b, bias, absmax)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    if a_mn_major:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn_major:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert K == Kb, "inner dimensions differ: %d vs %d" % (K, Kb)
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=a.device)
    assert out.stride(1) == 1
    pre = torch.empty((M, N), dtype=torch.bfloat16, device=a.device) if want_preact else None
    if act == ACT_GELU_GRAD:
        assert aux is not None and aux.shape == (M, N) and aux.dtype == torch.bfloat16 and not want_preact
        assert aux.stride(1) == 1 and aux.stride(0) == out.stride(0)
        pre = aux
    if bias is not None:
        assert bias.dtype == torch.bfloat16 and bias.numel() == N
    rc = lib().cv_gemm_bf16(ptr(a), int(a_mn_major), a.stride(0), ptr(b), int(b_mn_major), b.stride(0),
                            ptr(out), int(out.dtype == torch.float32), out.stride(0), ptr(pre), ptr(bias), int(act),
                            ptr(absmax), M, N, K, block_n, *_drop3(dropout), stream_ptr())
    check(rc, "cv_gemm_bf16")
    return (out, pre) if want_preact else out


# ----------------------------------------------------------------------------------------------------
# abs-max LayerNorm
# ----------------------------------------------------------------------------------------------------
def new_scalars(n, device):
    """n zero-initialised fp32 scalars (abs-max accumulators must start at a non-negative value)."""
    return torch.zeros(n, dtype=torch.float32, device=device)


def absmax(x, out=None):
    require_cuda(x)
    x = x.contiguous()
    if out is None:
        out = torch.zeros(1, dtype=torch.float32, device=x.device)
    assert x.dtype in (torch.float32, torch.bfloat16)
    check(lib().cv_absmax(ptr(x), int(x.dtype == torch.bfloat16), x.numel(), ptr(out), stream_ptr()), "cv_absmax")
    return out


def layernorm_absmax_fwd(x, absmax_in, gamma, beta, eps, *, residual=None, out_dtype=torch.bfloat16,
                         absmax_out=None, save_stats=False):
    """x: [rows, cols] fp32|bf16 contiguous.  Returns (out, mean, rstd) (stats None unless save_stats)."""
    require_cuda(x, absmax_in, gamma, beta, residual)
    assert x.is_contiguous() and x.dim() == 2
    rows, cols = x.shape
    assert gamma.dtype == torch.bfloat16 and beta.dtype == torch.bfloat16
    out = torch.empty((rows, cols), dtype=out_dtype, device=x.device)
    mean = rstd = None
    if save_stats:
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.is_contiguous() and residual.shape == x.shape
    rc = lib().cv_layernorm_absmax_fwd(ptr(x), int(x.dtype == torch.bfloat16), ptr(absmax_in), ptr(gamma), ptr(beta),
                                       float(eps), ptr(residual), ptr(out), int(out_dtype == torch.bfloat16),
                                       ptr(absmax_out), ptr(mean), ptr(rstd), rows, cols, stream_ptr())
    check(rc, "cv_layernorm_absmax_fwd")
    return out, mean, rstd


def _drop3(dropout):
    if dropout is None or dropout[0] <= 0:
        return 0.0, 0, 0
    return float(dropout[0]), int(dropout[1]), int(dropout[2])


def dropout_mask(n, p, seed, site, device="cuda"):
    """Keep mask (uint8) of the first n elements of dropout site (seed, site) — what every fused dropout uses."""
    out = torch.empty(n, dtype=torch.uint8, device=device)
    check(lib().cv_dropout_mask(ptr(out), n, float(p), int(seed), int(site), stream_ptr()), "cv_dropout_mask")
    return out


def layernorm_absmax_bwd(x, dy, mean, rstd, gamma, *, dres=None, dx_dtype=torch.float32, dropout=None,
                         want_dxsum=False):
    """Returns (dx, dgamma, dbeta) [+ column sums of dx when want_dxsum (hidden size % 256 == 0)]."""
    require_cuda(x, dy, mean, rstd, gamma, dres)
    assert x.is_contiguous() and dy.is_contiguous()
    rows, cols = x.shape
    dx = torch.empty((rows, cols), dtype=dx_dtype, device=x.device)
    dgamma = torch.empty(cols, dtype=torch.bfloat16, device=x.device)
    dbeta = torch.empty(cols, dtype=torch.bfloat16, device=x.device)
    ws = torch.empty(lib().cv_layernorm_bwd_workspace_bytes(rows, cols) // 4, dtype=torch.float32, device=x.device)
    dxsum = torch.empty(cols, dtype=torch.bfloat16, device=x.device) if want_dxsum else None
    if dres is not None:
        assert dres.dtype == torch.float32 and dres.is_contiguous()
    rc = lib().cv_layernorm_absmax_bwd(ptr(x), int(x.dtype == torch.bfloat16), ptr(dy),
                                       int(dy.dtype == torch.bfloat16), ptr(mean), ptr(rstd), ptr(gamma), ptr(dres),
                                       ptr(dx), int(dx_dtype == torch.bfloat16), ptr(dgamma), ptr(dbeta), ptr(ws),
                                       rows, cols, *_drop3(dropout), ptr(dxsum), stream_ptr())
    check(rc, "cv_layernorm_absmax_bwd")
    if want_dxsum:
        return dx, dgamma, dbeta, dxsum
    return dx, dgamma, dbeta


# ----------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------
def attn_fwd(q, k, v, heads, *, sep=0, want_lse=False, dropout=None):
    """q: [b, sq, heads*64] view, k/v: [b, sk, heads*64] views (last dim contiguous, bf16).
    Returns ctx [b, sq, heads*64] bf16 (and lse [b, heads, sq] fp32; and the keep-bit tensor when dropout is on)."""
    require_cuda(q, k, v)
    b, sq, hq = q.shape
    sk = k.shape[1]
    assert q.stride(2) == 1 and k.stride(2) == 1 and v.stride(2) == 1
    assert hq == heads * 64 and k.shape[2] == hq and v.shape == k.shape
    out = torch.empty((b, sq, hq), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((b, heads, sq), dtype=torch.float32, device=q.device) if want_lse else None
    dp, dseed, dsite = _drop3(dropout)
    mask = None
    if dp > 0:
        # keep bits in two layouts: [0] key-major [b, heads, key (padded to 128), query block, 4 x 32 queries] for the
        # backward, [1] query-major [b, heads, query (padded), key block, 4 x 32 keys] for the forward kernel
        mask = torch.empty((2, b, heads, ((sk + 127) // 128) * ((sq + 127) // 128) * 128, 4), dtype=torch.int32,
                           device=q.device)
    rc = lib().cv_attn_fwd(ptr(q), q.stride(1), q.stride(0), ptr(k), k.stride(1), k.stride(0), ptr(v), v.stride(1),
                           v.stride(0), ptr(out), out.stride(1), out.stride(0), ptr(lse), b, heads, 64, sq, sk,
                           int(sep), dp, dseed, dsite, ptr(mask), stream_ptr())
    check(rc, "cv_attn_fwd")
    if dp > 0:
        return (out, lse, mask) if want_lse else (out, mask)
    return (out, lse) if want_lse else out


def attn_bwd(q, k, v, out, d_out, lse, heads, *, sep=0, dropout_p=0.0, drop_mask=None):
    """Backward of attn_fwd for sq == sk.  Returns dqkv [b, s, 3*heads*64] bf16 (dQ | dK | dV)."""
    require_cuda(q, k, v, out, d_out, lse)
    b, s, h = q.shape
    assert k.shape[1] == s, "attention backward needs sq == sk"
    assert out.is_contiguous() and d_out.is_contiguous() and d_out.dtype == torch.bfloat16
    dqkv = torch.empty((b, s, 3 * h), dtype=torch.bfloat16, device=q.device)
    ws = torch.empty(lib().cv_attn_bwd_workspace_bytes(b, heads, 64, s) // 4, dtype=torch.float32, device=q.device)
    rc = lib().cv_attn_bwd(ptr(q), q.stride(1), q.stride(0), ptr(k), k.stride(1), k.stride(0), ptr(v), v.stride(1),
                           v.stride(0), ptr(out), ptr(d_out), ptr(lse), ptr(dqkv), ptr(ws), b, heads, 64, s, int(sep),
                           float(dropout_p), ptr(drop_mask), stream_ptr())
    check(rc, "cv_attn_bwd")
    return dqkv


def attn_sparse_fwd(q, k, v, heads, pivot_idx, query_window, key_window_times, *, want_lse=False, dropout=None):
    """Sparse TRAINING attention (mpu/sparse_transformer.py:675-725): q, k, v [b, s, heads*64] bf16 views,
    pivot_idx int64 [b, n_piv].  Returns ctx [b, s, heads*64] bf16 (and lse [b, heads, s] fp32; and the keep-bit tensor
    when dropout = (p, seed, site) has p > 0 — int32 [cv_attn_sparse_drop_mask_words()], layout in the C header)."""
    require_cuda(q, k, v, pivot_idx)
    b, s, h = q.shape
    n_piv = pivot_idx.shape[1]
    assert q.stride(2) == 1 and k.stride(2) == 1 and v.stride(2) == 1 and h == heads * 64
    assert pivot_idx.dtype == torch.int64 and pivot_idx.shape[0] == b
    pivot_idx = pivot_idx.contiguous()
    out = torch.empty((b, s, h), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((b, heads, s), dtype=torch.float32, device=q.device) if want_lse else None
    ws = torch.empty(lib().cv_attn_sparse_workspace_bytes(b, heads, 64, n_piv), dtype=torch.uint8, device=q.device)
    dp, dseed, dsite = _drop3(dropout)
    mask = None
    if dp > 0:
        words = lib().cv_attn_sparse_drop_mask_words(b, heads, s, n_piv, int(query_window), int(key_window_times))
        check(words if words < 0 else 0, "cv_attn_sparse_drop_mask_words")
        mask = torch.empty(words, dtype=torch.int32, device=q.device)
    rc = lib().cv_attn_sparse_fwd(
        ptr(q), q.stride(1), q.stride(0), ptr(k), k.stride(1), k.stride(0), ptr(v), v.stride(1), v.stride(0),
        ptr(pivot_idx), ptr(out), out.stride(1), out.stride(0), ptr(lse), ptr(ws), b, heads, 64, s, n_piv,
        int(query_window), int(key_window_times), dp, dseed, dsite, ptr(mask), stream_ptr())
    check(rc, "cv_attn_sparse_fwd")
    if mask is not None:
        return (out, lse, mask) if want_lse else (out, mask)
    return (out, lse) if want_lse else out


def attn_sparse_bwd(q, k, v, out, d_out, lse, heads, pivot_idx, query_window, key_window_times, *, dropout_p=0.0,
                    drop_mask=None):
    """Backward of attn_sparse_fwd (dropout_p > 0: drop_mask is the keep-bit tensor it returned).
    Returns dqkv [b, s, 3*heads*64] bf16 (dQ | dK | dV)."""
    require_cuda(q, k, v, out, d_out, lse, pivot_idx)
    b, s, h = q.shape
    n_piv = pivot_idx.shape[1]
    assert out.is_contiguous() and d_out.is_contiguous() and d_out.dtype == torch.bfloat16
    pivot_idx = pivot_idx.contiguous()
    dqkv = torch.empty((b, s, 3 * h), dtype=torch.bfloat16, device=q.device)
    ws = torch.empty(lib().cv_attn_sparse_bwd_workspace_bytes(b, heads, 64, s, n_piv), dtype=torch.uint8,
                     device=q.device)
    dp = float(dropout_p) if dropout_p > 0 else 0.0
    if dp > 0:
        require_cuda(drop_mask)
    rc = lib().cv_attn_sparse_bwd(
        ptr(q), q.stride(1), q.stride(0), ptr(k), k.stride(1), k.stride(0), ptr(v), v.stride(1), v.stride(0),
        ptr(pivot_idx), ptr(out), ptr(d_out), ptr(lse), ptr(dqkv), ptr(ws), b, heads, 64, s, n_piv,
        int(query_window), int(key_window_times), dp, ptr(drop_mask), stream_ptr())
    check(rc, "cv_attn_sparse_bwd")
    return dqkv


# ----------------------------------------------------------------------------------------------------
# embedding, cross-entropy, small backward helpers
# ----------------------------------------------------------------------------------------------------
def embed_fwd(ids, pos, wte, wpe, absmax_out=None, dropout=None):
    require_cuda(ids, pos, wte, wpe)
    ids = ids.contiguous().view(-1)
    pos = pos.contiguous().view(-1)
    assert ids.dtype == torch.int64 and pos.dtype == torch.int64 and ids.numel() == pos.numel()
    assert wte.dtype == torch.bfloat16 and wpe.dtype == torch.bfloat16 and wte.is_contiguous() and wpe.is_contiguous()
    h = wte.shape[1]
    out = torch.empty((ids.numel(), h), dtype=torch.float32, device=wte.device)
    check(lib().cv_embed_fwd(ptr(ids), ptr(pos), ptr(wte), ptr(wpe), ptr(out), ptr(absmax_out), ids.numel(), h,
                             *_drop3(dropout), stream_ptr()), "cv_embed_fwd")
    return out


def embed_bwd(ids, pos, dx, dwte, dwpe, dropout=None):
    """Accumulates into dwte / dwpe (bf16, contiguous)."""
    require_cuda(ids, pos, dx, dwte, dwpe)
    ids = ids.contiguous().view(-1)
    pos = pos.contiguous().view(-1)
    assert dx.dtype == torch.float32 and dx.is_contiguous()
    check(lib().cv_embed_bwd(ptr(ids), ptr(pos), ptr(dx), ptr(dwte), ptr(dwpe), ids.numel(), dwte.shape[1],
                             *_drop3(dropout), stream_ptr()), "cv_embed_bwd")


def cross_entropy_fwd(logits, target):
    """logits: [rows, V] fp32 (last dim contiguous); target int64 [rows].  Returns (loss, row_max, row_sum)."""
    require_cuda(logits, target)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    rows, V = logits.shape
    target = target.contiguous().view(-1)
    assert target.numel() == rows and target.dtype == torch.int64
    loss = torch.empty(rows, dtype=torch.float32, device=logits.device)
    rmax = torch.empty_like(loss)
    rsum = torch.empty_like(loss)
    check(lib().cv_cross_entropy_fwd(ptr(logits), logits.stride(0), ptr(target), ptr(loss), ptr(rmax), ptr(rsum), rows,
                                     V, stream_ptr()), "cv_cross_entropy_fwd")
    return loss, rmax, rsum


def cross_entropy_bwd(logits, target, rmax, rsum, grad_loss):
    require_cuda(logits, target, grad_loss)
    rows, V = logits.shape
    target = target.contiguous().view(-1)
    grad_loss = grad_loss.contiguous().view(-1).float()
    ldd = (V + 7) // 8 * 8
    dl = torch.empty((rows, ldd), dtype=torch.bfloat16, device=logits.device)
    check(lib().cv_cross_entropy_bwd(ptr(logits), logits.stride(0), ptr(target), ptr(rmax), ptr(rsum), ptr(grad_loss),
                                     ptr(dl), ldd, rows, V, stream_ptr()), "cv_cross_entropy_bwd")
    return dl[:, :V]


def vocab_logprob(h, w, target, v_begin=0, v_end=None):
    """log_softmax(h @ w[v_begin:v_end]^T)[m, target[m] - v_begin] for every row m, without materialising the logits:
    h bf16 [M, K], w bf16 [V, K] (the tied word embedding), target int64 [M] (absolute vocabulary ids; one outside
    [v_begin, v_end) gives -inf).  Returns fp32 [M]."""
    require_cuda(h, w, target)
    assert h.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and h.dim() == 2 and w.dim() == 2
    assert h.stride(1) == 1 and w.stride(1) == 1 and h.shape[1] == w.shape[1]
    M, K = h.shape
    v_end = w.shape[0] if v_end is None else v_end
    assert 0 <= v_begin < v_end <= w.shape[0], "vocabulary window [%d, %d) outside [0, %d)" % (v_begin, v_end,
                                                                                            w.shape[0])
    target = target.contiguous().view(-1)
    assert target.dtype == torch.int64 and target.numel() == M
    out = torch.empty(M, dtype=torch.float32, device=h.device)
    if M == 0:
        return out
    ws = torch.empty(lib().cv_vocab_logprob_workspace_bytes(M, v_begin, v_end) // 4, dtype=torch.float32,
                     device=h.device)
    check(lib().cv_vocab_logprob(ptr(h), h.stride(0), ptr(w), w.stride(0), ptr(target), ptr(out), ptr(ws), M, K,
                                 int(v_begin), int(v_end), stream_ptr()), "cv_vocab_logprob")
    return out


# Byte budget of one bf16 dlogits chunk [M, width] in the fused cross-entropy backward (vocab_xent_bwd): the largest
# tensor it allocates.  256 MiB holds the whole 58240-column vocabulary for up to 2304 rows (2 x 1088 tokens fit).
XENT_CHUNK_BYTES = 256 << 20


def xent_chunks(M, V, chunk_bytes=None):
    """Column windows [(v0, v1), ...] of the fused backward, in order and covering [0, V): one window when the bf16
    dlogits of all V columns (rows padded to 8 columns) fit `chunk_bytes` (default XENT_CHUNK_BYTES), else windows
    of the largest multiple of 256 columns that fits (at least 256), the last one taking the remainder."""
    budget = XENT_CHUNK_BYTES if chunk_bytes is None else int(chunk_bytes)
    if M * ((V + 7) // 8 * 8) * 2 <= budget:
        return [(0, V)]
    width = max(256, budget // (2 * M) // 256 * 256)
    return [(v0, min(V, v0 + width)) for v0 in range(0, V, width)]


def add_f32(dst, src):
    """dst += src (fp32, contiguous, same number of elements, a multiple of 4)."""
    require_cuda(dst, src)
    assert dst.dtype == torch.float32 and src.dtype == torch.float32 and dst.is_contiguous() and src.is_contiguous()
    assert dst.numel() == src.numel()
    check(lib().cv_add_f32(ptr(dst), ptr(src), dst.numel(), stream_ptr()), "cv_add_f32")
    return dst


def _xent_args(h, w, target):
    require_cuda(h, w, target)
    assert h.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and h.dim() == 2 and w.dim() == 2
    assert h.stride(1) == 1 and w.stride(1) == 1 and h.shape[1] == w.shape[1]
    target = target.contiguous().view(-1)
    assert target.dtype == torch.int64 and target.numel() == h.shape[0]
    return target


def vocab_xent_fwd(h, w, target):
    """Per-token cross-entropy over the whole vocabulary without logits in memory: h bf16 [M, K] (the final
    LayerNorm's output), w bf16 [V, K] (the tied word embedding), target int64 [M].  Returns (loss, lse), fp32 [M]:
    loss = lse - h . w[target], lse = logsumexp(h @ w^T) per row, from the same fp32 GEMM accumulators the logits
    route rounds; only the order of the sum of exponentials differs.  A target outside [0, V) gives loss NaN.  Equal
    inputs give equal bits."""
    target = _xent_args(h, w, target)
    M, K = h.shape
    V = w.shape[0]
    loss = torch.empty(M, dtype=torch.float32, device=h.device)
    lse = torch.empty(M, dtype=torch.float32, device=h.device)
    if M == 0:
        return loss, lse
    ws = torch.empty(lib().cv_vocab_xent_workspace_bytes(M, V) // 4, dtype=torch.float32, device=h.device)
    check(lib().cv_vocab_xent_fwd(ptr(h), h.stride(0), ptr(w), w.stride(0), ptr(target), ptr(loss), ptr(lse), ptr(ws),
                                  M, K, V, stream_ptr()), "cv_vocab_xent_fwd")
    return loss, lse


def vocab_xent_dlogits(h, w, target, lse, grad_loss, v_begin, v_end, out=None):
    """bf16 [M, v_end - v_begin] = grad_loss[m] * (softmax(h @ w^T)[m, v] - [v == target[m]]) for v in
    [v_begin, v_end), recomputing the logits of the window; lse from vocab_xent_fwd.  `out` (bf16 [M, >= width],
    last dim contiguous, even row stride) receives it in its first v_end - v_begin columns."""
    target = _xent_args(h, w, target)
    M, K = h.shape
    assert 0 <= v_begin < v_end <= w.shape[0], "vocabulary window [%d, %d) outside [0, %d)" % (v_begin, v_end,
                                                                                            w.shape[0])
    n = v_end - v_begin
    if out is None:
        out = torch.empty((M, (n + 7) // 8 * 8), dtype=torch.bfloat16, device=h.device)[:, :n]
    require_cuda(lse, grad_loss, out)
    assert out.dtype == torch.bfloat16 and out.stride(1) == 1 and out.shape[0] == M and out.shape[1] >= n
    assert lse.dtype == torch.float32 and lse.is_contiguous() and lse.numel() == M
    grad_loss = grad_loss.reshape(-1).float().contiguous()
    assert grad_loss.numel() == M
    check(lib().cv_vocab_xent_dlogits(ptr(h), h.stride(0), ptr(w), w.stride(0), ptr(target), ptr(lse), ptr(grad_loss),
                                      ptr(out), out.stride(0), M, K, int(v_begin), int(v_end), stream_ptr()),
          "cv_vocab_xent_dlogits")
    return out[:, :n]


def vocab_xent_bwd(h, w, target, lse, grad_loss, chunk_bytes=None):
    """Backward of vocab_xent_fwd, never holding [M, V]: for each column window [v0, v1) of xent_chunks(M, V,
    chunk_bytes), D = vocab_xent_dlogits (bf16, as the logits route's dlogits), dW[v0:v1] = D^T h (the wgrad GEMM,
    written in place) and dH += D w[v0:v1] (the dgrad GEMM).  Returns (dH bf16 [M, K], dW bf16 [V, K]).  With one
    window dH is the dgrad GEMM's bf16 output, as in the logits route; with several it is summed in fp32 in window
    order and rounded once.  Equal inputs and budget give equal bits."""
    target = _xent_args(h, w, target)
    M, K = h.shape
    V = w.shape[0]
    chunks = xent_chunks(M, V, chunk_bytes)
    widest = max(v1 - v0 for v0, v1 in chunks)
    d = torch.empty((M, (widest + 7) // 8 * 8), dtype=torch.bfloat16, device=h.device)
    dw = torch.empty((V, K), dtype=torch.bfloat16, device=h.device)
    if len(chunks) == 1:
        dc = vocab_xent_dlogits(h, w, target, lse, grad_loss, 0, V, out=d)
        dh = gemm(dc, w, b_mn_major=True)
        gemm(dc, h, a_mn_major=True, b_mn_major=True, out=dw)
        return dh, dw
    dh = torch.empty((M, K), dtype=torch.float32, device=h.device)
    part = torch.empty_like(dh)
    for i, (v0, v1) in enumerate(chunks):
        dc = vocab_xent_dlogits(h, w, target, lse, grad_loss, v0, v1, out=d)
        gemm(dc, h, a_mn_major=True, b_mn_major=True, out=dw[v0:v1])
        gemm(dc, w[v0:v1], b_mn_major=True, out_dtype=torch.float32, out=dh if i == 0 else part)
        if i > 0:
            add_f32(dh, part)
    del d, dc, part
    return dh.to(torch.bfloat16), dw


def gelu_bwd(pre, dact):
    require_cuda(pre, dact)
    assert pre.is_contiguous() and dact.is_contiguous() and pre.dtype == torch.bfloat16 and dact.dtype == torch.bfloat16
    out = torch.empty_like(pre)
    check(lib().cv_gelu_bwd(ptr(pre), ptr(dact), ptr(out), pre.numel(), stream_ptr()), "cv_gelu_bwd")
    return out


def colsum(dy):
    """bias gradient: sum over rows of a [rows, cols] bf16 matrix -> [cols] bf16."""
    require_cuda(dy)
    assert dy.dim() == 2 and dy.stride(1) == 1 and dy.dtype == torch.bfloat16
    rows, cols = dy.shape
    out = torch.empty(cols, dtype=torch.bfloat16, device=dy.device)
    ws = torch.empty(lib().cv_colsum_workspace_bytes(cols) // 4, dtype=torch.float32, device=dy.device)
    check(lib().cv_colsum_bf16(ptr(dy), dy.stride(0), ptr(out), ptr(ws), rows, cols, stream_ptr()), "cv_colsum_bf16")
    return out


# ----------------------------------------------------------------------------------------------------
# decode (weight-streaming) kernels
# ----------------------------------------------------------------------------------------------------
def _decode_linear(name, x, w, bias, act, out_dtype, absmax, out):
    require_cuda(x, w, bias, absmax)
    M, K = x.shape
    N = w.shape[0]
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x.stride(1) == 1 and w.stride(1) == 1
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
    rc = getattr(lib(), name)(ptr(x), x.stride(0), ptr(w), w.stride(0), ptr(bias), ptr(out), out.stride(0),
                              int(out.dtype == torch.float32), int(act), ptr(absmax), M, N, K, stream_ptr())
    check(rc, name)
    return out


def linear_small_m(x, w, bias=None, *, act=ACT_NONE, out_dtype=torch.bfloat16, absmax=None, out=None):
    """y = x @ w^T + bias for 1 <= M <= 16 rows (x: [M,K] bf16, w: [N,K] bf16)."""
    return _decode_linear("cv_linear_small_m", x, w, bias, act, out_dtype, absmax, out)


def linear_mid_m(x, w, bias=None, *, act=ACT_NONE, out_dtype=torch.bfloat16, absmax=None, out=None):
    """y = x @ w^T + bias for 17 <= M <= 64 rows (x: [M,K] bf16, w: [N,K] bf16)."""
    return _decode_linear("cv_linear_mid_m", x, w, bias, act, out_dtype, absmax, out)


def attn_decode(qkv, cache, heads, *, cur_len=None, cur_len_dev=None, nsplit=1, out=None, workspace=None,
                row_pad=None):
    """qkv: [b, 3h] bf16; cache: [b, max_len, 2h] bf16 (K|V); appends the new token at cur_len and returns
    the attention context [b, h] bf16.  row_pad (int32 [b] on the device, 0 <= row_pad[i] <= cur_len): row i holds
    cur_len - row_pad[i] cached tokens and appends there."""
    require_cuda(qkv, cache, row_pad)
    b, h3 = qkv.shape
    h = h3 // 3
    assert qkv.is_contiguous() and cache.stride(2) == 1 and cache.stride(1) == 2 * h and cache.shape[2] == 2 * h
    if out is None:
        out = torch.empty((b, h), dtype=torch.bfloat16, device=qkv.device)
    if nsplit > 1 and workspace is None:
        workspace = torch.empty(lib().cv_attn_decode_workspace_bytes(b, heads, nsplit) // 4, dtype=torch.float32,
                                device=qkv.device)
    cl = -1 if cur_len is None else int(cur_len)
    if row_pad is not None:
        assert row_pad.dtype == torch.int32 and row_pad.is_contiguous() and row_pad.numel() == b
    rc = lib().cv_attn_decode(ptr(qkv), ptr(cache), cache.stride(0), ptr(cur_len_dev), cl, ptr(row_pad), ptr(out),
                              ptr(workspace), b, heads, 64, cache.shape[1], nsplit, stream_ptr())
    check(rc, "cv_attn_decode")
    return out


ATTN_CHUNK_MAX = 64      # tokens per row of one cv_attn_chunk_ragged call


def attn_chunk_nsplit(b, heads, keys, device):
    """Key splits per (row, head) for cv_attn_chunk_ragged: about four CTAs per SM in all (a CTA walks its key range
    one 64-key tile at a time, so one or two CTAs per SM leave HBM idle), at least 128 keys each."""
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    return max(1, min(16, -(-4 * sms // (b * heads)), -(-keys // 128)))


def attn_chunk_ragged(qkv, cache, heads, cur_len, row_pad=None, *, nsplit=None, out=None, workspace=None):
    """Attention of a chunk of n new tokens per row against that row's cached prefix, with the chunk's K|V appended
    (cv_attn_chunk_ragged).  qkv: [b, n, 3h] bf16 (the QKV GEMM output, read in place); cache: [b, max_len, 2h] bf16
    (K|V, row stride 2h); row_pad: int32 [b] on the device or None — row i holds cur_len - row_pad[i] cached tokens,
    query j of row i attends keys 0 .. cur_len - row_pad[i] + j, and the chunk is written at slots
    cur_len - row_pad[i] ... onwards.  Returns the context [b, n, h] bf16."""
    require_cuda(qkv, cache, row_pad)
    b, n, h3 = qkv.shape
    h = h3 // 3
    assert qkv.dtype == torch.bfloat16 and cache.dtype == torch.bfloat16 and qkv.is_contiguous()
    assert cache.shape[0] == b and cache.stride(2) == 1 and cache.stride(1) == 2 * h and cache.shape[2] == 2 * h
    if row_pad is not None:
        assert row_pad.dtype == torch.int32 and row_pad.is_contiguous() and row_pad.numel() == b
    if nsplit is None:
        nsplit = attn_chunk_nsplit(b, heads, int(cur_len) + n, qkv.device)
    if out is None:
        out = torch.empty((b, n, h), dtype=torch.bfloat16, device=qkv.device)
    if nsplit > 1 and workspace is None:
        workspace = torch.empty(lib().cv_attn_chunk_workspace_bytes(b, heads, n, nsplit) // 4, dtype=torch.float32,
                                device=qkv.device)
    rc = lib().cv_attn_chunk_ragged(ptr(qkv), ptr(cache), cache.stride(0), int(cur_len), ptr(row_pad), ptr(out),
                                    ptr(workspace), b, n, heads, 64, cache.shape[1], nsplit, stream_ptr())
    check(rc, "cv_attn_chunk_ragged")
    return out


def attn_decode_shared(qkv, prefix, suffix, heads, prefix_len, *, s=None, s_dev=None, nsplit=None, out=None,
                       workspace=None):
    """Decode attention for rows that share a prompt (cv_attn_decode_shared).  qkv: [b, 3h] bf16; prefix:
    [groups, max_len, 2h] bf16 (K|V of every group's prompt, prefix_len tokens each; read only); suffix:
    [b, s_max, 2h] bf16 (K|V of every row's generated tokens).  Row r of group r // (b // groups) attends
    prefix[g, :prefix_len], suffix[r, :s] and its new key, and its k|v is written at suffix[r, s].  s from the host,
    or from s_dev (int32 [1] on the device, read when the kernel runs).  Returns the context [b, h] bf16."""
    require_cuda(qkv, prefix, suffix, s_dev)
    b, h3 = qkv.shape
    h = h3 // 3
    groups = prefix.shape[0]
    assert qkv.dtype == prefix.dtype == suffix.dtype == torch.bfloat16 and qkv.is_contiguous()
    for c in (prefix, suffix):
        assert c.stride(2) == 1 and c.stride(1) == 2 * h and c.shape[2] == 2 * h
    assert suffix.shape[0] == b and (s_dev is None or s_dev.dtype == torch.int32)
    if nsplit is None:
        nsplit = attn_chunk_nsplit(groups, heads, prefix_len, qkv.device)
    if out is None:
        out = torch.empty((b, h), dtype=torch.bfloat16, device=qkv.device)
    if workspace is None:
        workspace = torch.empty(lib().cv_attn_shared_workspace_bytes(b, heads, nsplit) // 4, dtype=torch.float32,
                                device=qkv.device)
    rc = lib().cv_attn_decode_shared(ptr(qkv), ptr(prefix), prefix.stride(0), int(prefix_len), prefix.shape[1],
                                     ptr(suffix), suffix.stride(0), ptr(s_dev), -1 if s is None else int(s),
                                     suffix.shape[1], ptr(out), ptr(workspace), b, groups, heads, 64, nsplit,
                                     stream_ptr())
    check(rc, "cv_attn_decode_shared")
    return out


def sparse_plan(is_txt, cur_len_dev, num_layers, window, num_pivot, max_sequence_length, seed_dev, idx, n_dev, err):
    """Index plan of one sparse decode step for every layer (cv_sparse_plan).  is_txt: uint8 [b, max_len]; idx: int32
    [num_layers, b, nmax] (written); n_dev, err: int32 [1]; seed_dev: int64 [1]."""
    require_cuda(is_txt, cur_len_dev, seed_dev, idx, n_dev, err)
    assert is_txt.dtype == torch.uint8 and is_txt.stride(1) == 1 and idx.dtype == torch.int32 and idx.is_contiguous()
    assert cur_len_dev.dtype == torch.int32 and n_dev.dtype == torch.int32 and seed_dev.dtype == torch.int64
    L, b, nmax = idx.shape
    assert L == num_layers and is_txt.shape[0] == b
    check(lib().cv_sparse_plan(ptr(is_txt), is_txt.stride(0), ptr(cur_len_dev), int(num_layers), b, int(window),
                               int(num_pivot), int(max_sequence_length), ptr(seed_dev), ptr(idx), nmax, ptr(n_dev),
                               ptr(err), stream_ptr()), "cv_sparse_plan")


def attn_decode_gather(qkv, cache, heads, cur_len_dev, idx, n_dev, *, nsplit=1, out=None, workspace=None):
    """attn_decode over the key list idx [b, nmax] int32 (first *n_dev entries; it contains the new token's position)."""
    require_cuda(qkv, cache, idx, n_dev, cur_len_dev)
    b, h3 = qkv.shape
    h = h3 // 3
    assert qkv.is_contiguous() and cache.stride(2) == 1 and cache.stride(1) == 2 * h and cache.shape[2] == 2 * h
    assert idx.dtype == torch.int32 and idx.shape[0] == b and idx.stride(1) == 1
    if out is None:
        out = torch.empty((b, h), dtype=torch.bfloat16, device=qkv.device)
    if nsplit > 1 and workspace is None:
        workspace = torch.empty(lib().cv_attn_decode_workspace_bytes(b, heads, nsplit) // 4, dtype=torch.float32,
                                device=qkv.device)
    rc = lib().cv_attn_decode_gather(ptr(qkv), ptr(cache), cache.stride(0), ptr(cur_len_dev), ptr(idx), idx.stride(0),
                                     ptr(n_dev), ptr(out), ptr(workspace), b, heads, 64, cache.shape[1], nsplit,
                                     stream_ptr())
    check(rc, "cv_attn_decode_gather")
    return out


def _decode_ln_pair(name, res_in, gemm_out, absmax_gemm, post, pre, eps, want_res_out):
    require_cuda(res_in, gemm_out)
    M, K = res_in.shape
    assert res_in.dtype == torch.float32 and res_in.is_contiguous()
    y = torch.empty_like(res_in) if want_res_out else None
    xn = torch.empty((M, K), dtype=torch.bfloat16, device=res_in.device)
    gp, bp = post if post is not None else (None, None)
    rc = getattr(lib(), name)(ptr(res_in), ptr(gemm_out), ptr(absmax_gemm), ptr(gp), ptr(bp), ptr(pre[0]),
                              ptr(pre[1]), float(eps), ptr(y), ptr(xn), M, K, stream_ptr())
    check(rc, name)
    return y, xn


def ln_pair_small_m(res_in, gemm_out, absmax_gemm, post, pre, eps, *, want_res_out=True):
    """y = res_in + LN_post(gemm_out) (gemm_out may be None), xn = LN_pre(y).  post/pre: (gamma, beta) bf16.
    1 <= M <= 16 rows.  Returns (y fp32 or None, xn bf16)."""
    return _decode_ln_pair("cv_ln_pair_small_m", res_in, gemm_out, absmax_gemm, post, pre, eps, want_res_out)


def ln_pair_mid_m(res_in, gemm_out, absmax_gemm, post, pre, eps, *, want_res_out=True):
    """ln_pair_small_m for 17 <= M <= 64 rows."""
    return _decode_ln_pair("cv_ln_pair_mid_m", res_in, gemm_out, absmax_gemm, post, pre, eps, want_res_out)


# sequences per decode step: up to DECODE_SMALL_MAX_BATCH the *_small_m kernels, up to DECODE_MAX_BATCH the *_mid_m ones
DECODE_SMALL_MAX_BATCH = 16
DECODE_MAX_BATCH = 64
LN_PAIR_MID_MAX_HIDDEN = 2560      # cv_ln_pair_mid_m keeps a row in the registers of 128 threads


def decode_batch_supported(b, hidden):
    """True if the per-operation decode kernels cover b sequences per step at this hidden size."""
    return b <= DECODE_SMALL_MAX_BATCH or (b <= DECODE_MAX_BATCH and hidden <= LN_PAIR_MID_MAX_HIDDEN)


def valid_ranges(invalid, vocab):
    """Complement of a list of [lo, hi) index pairs inside [0, vocab) as a sorted list of [lo, hi) pairs."""
    inv = sorted((max(0, int(a)), min(vocab, int(z))) for a, z in invalid)
    out, cur = [], 0
    for a, z in inv:
        if a > cur:
            out.append((cur, a))
        cur = max(cur, z)
    if cur < vocab:
        out.append((cur, vocab))
    return out


def sample_topk(logits, temperature, top_k, valid, *, seed=0, seed_dev=None, step=None, next_ids=None, out_tokens=None,
                score_acc=None, pos=None, cur_len=None, done=None, want_probs=False, top_p=0.0):
    """Sampling tail of generation/sampling.py:157-183 in one kernel.  logits fp32 [b, V] (unchanged);
    valid: list of [lo, hi) vocabulary ranges (<= 4).  top_p > 0 adds the nucleus filter after top-k.
    Returns (next_ids int64 [b], probs or None)."""
    import ctypes
    require_cuda(logits, seed_dev, step, next_ids, out_tokens, score_acc, pos, cur_len, done)
    b, V = logits.shape
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    if not 1 <= len(valid) <= 4:
        raise _lib.CogViewB200Error("cv_sample_topk takes 1..4 valid vocabulary ranges, got %r" % (valid,))
    if next_ids is None:
        next_ids = torch.empty(b, dtype=torch.int64, device=logits.device)
    if (step is not None or cur_len is not None) and done is None:
        done = torch.zeros(1, dtype=torch.int32, device=logits.device)
    probs = torch.empty((b, logits.stride(0)), dtype=torch.float32, device=logits.device) if want_probs else None
    flat = (ctypes.c_int * (2 * len(valid)))(*[int(x) for r in valid for x in r])
    rc = lib().cv_sample_topk(ptr(logits), logits.stride(0), b, V, float(temperature), int(top_k), flat, len(valid),
                              int(seed) & 0xFFFFFFFFFFFFFFFF, ptr(seed_dev), ptr(step), ptr(next_ids), ptr(out_tokens),
                              0 if out_tokens is None else out_tokens.stride(0), ptr(score_acc), ptr(pos), ptr(cur_len),
                              ptr(done), ptr(probs), float(top_p), stream_ptr())
    check(rc, "cv_sample_topk")
    return next_ids, (probs[:, :V] if want_probs else None)


# ----------------------------------------------------------------------------------------------------
# VQ-VAE kernels (NHWC bf16 activations)
# ----------------------------------------------------------------------------------------------------
def conv2d_k4s2(x, w_packed, bias, relu):
    """x: [B, H, W, Cin] bf16 NHWC; w_packed: [16, Cout, Cin] bf16 -> [B, H/2, W/2, Cout] bf16."""
    require_cuda(x, w_packed, bias)
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[1]
    assert x.is_contiguous() and w_packed.is_contiguous() and x.dtype == torch.bfloat16
    y = torch.empty((B, H // 2, W // 2, Cout), dtype=torch.bfloat16, device=x.device)
    check(lib().cv_conv2d_k4s2(ptr(x), ptr(w_packed), ptr(bias), ptr(y), B, H, W, Cin, Cout, int(relu), stream_ptr()),
          "cv_conv2d_k4s2")
    return y


def conv_transpose2d_k4s2(x, w_packed, bias, relu):
    """x: [B, H, W, Cin] bf16 NHWC; w_packed: [16, Cout, Cin] bf16 -> [B, 2H, 2W, Cout] bf16."""
    require_cuda(x, w_packed, bias)
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[1]
    assert x.is_contiguous() and w_packed.is_contiguous() and x.dtype == torch.bfloat16
    y = torch.empty((B, 2 * H, 2 * W, Cout), dtype=torch.bfloat16, device=x.device)
    check(lib().cv_conv_transpose2d_k4s2(ptr(x), ptr(w_packed), ptr(bias), ptr(y), B, H, W, Cin, Cout, int(relu),
                                         stream_ptr()), "cv_conv_transpose2d_k4s2")
    return y


def im2col_k4s2_c3(img):
    """img: [B, 3, H, W] fp32 NCHW -> [B*(H/2)*(W/2), 64] bf16 patches (48 used)."""
    require_cuda(img)
    B, C, H, W = img.shape
    assert C == 3 and img.dtype == torch.float32 and img.is_contiguous()
    out = torch.empty((B * (H // 2) * (W // 2), 64), dtype=torch.bfloat16, device=img.device)
    check(lib().cv_im2col_k4s2_c3(ptr(img), ptr(out), B, H, W, stream_ptr()), "cv_im2col_k4s2_c3")
    return out


def vq_split3(z):
    require_cuda(z)
    rows, dim = z.shape
    assert z.dtype == torch.float32 and z.is_contiguous()
    out = torch.empty((rows, 3 * dim), dtype=torch.bfloat16, device=z.device)
    check(lib().cv_vq_split3(ptr(z), ptr(out), rows, dim, stream_ptr()), "cv_vq_split3")
    return out


def vq_argmin(scores, e2, z, codebook, margin=1e-4):
    require_cuda(scores, e2, z, codebook)
    rows, n_embed = scores.shape
    assert scores.dtype == torch.float32 and scores.stride(1) == 1 and codebook.is_contiguous() and z.is_contiguous()
    idx = torch.empty(rows, dtype=torch.int64, device=scores.device)
    check(lib().cv_vq_argmin(ptr(scores), scores.stride(0), ptr(e2), ptr(z), ptr(codebook), ptr(idx), rows, n_embed,
                             codebook.shape[1], float(margin), stream_ptr()), "cv_vq_argmin")
    return idx


def vq_lookup(idx, codebook, want_bf16=True, want_f32=False):
    require_cuda(idx, codebook)
    idx = idx.contiguous().view(-1)
    rows, dim = idx.numel(), codebook.shape[1]
    ob = torch.empty((rows, dim), dtype=torch.bfloat16, device=idx.device) if want_bf16 else None
    of = torch.empty((rows, dim), dtype=torch.float32, device=idx.device) if want_f32 else None
    check(lib().cv_vq_lookup(ptr(idx), ptr(codebook), ptr(ob), ptr(of), rows, dim, stream_ptr()), "cv_vq_lookup")
    return ob, of


def conv1x1_out3(x, w, bias, scale, shift):
    """x: [B, H, W, Cin] bf16 NHWC; w: [3, Cin] fp32 -> [B, 3, H, W] fp32 = (x.w + bias) * scale + shift."""
    require_cuda(x, w, bias, scale, shift)
    B, H, W, Cin = x.shape
    assert x.is_contiguous() and w.is_contiguous() and w.dtype == torch.float32
    out = torch.empty((B, 3, H, W), dtype=torch.float32, device=x.device)
    check(lib().cv_conv1x1_out3(ptr(x), ptr(w), ptr(bias), ptr(scale), ptr(shift), ptr(out), B, H, W, Cin,
                                stream_ptr()), "cv_conv1x1_out3")
    return out


def conv_k4s2_wgrad(s, g):
    """Weight gradient of a k4 s2 p1 convolution: s [B, h, w, M], g [B, 2h, 2w, N] bf16 NHWC -> fp32 [M, N, 4, 4],
    out[m, n, ky, kx] = sum_{b,y,x} s[b, y, x, m] g[b, 2y-1+ky, 2x-1+kx, n].  Conv2d: (s, g) = (dY, X) gives dW
    [Cout, Cin, 4, 4]; ConvTranspose2d: (s, g) = (X, dY) gives dW [Cin, Cout, 4, 4]."""
    require_cuda(s, g)
    B, h, w, M = s.shape
    N = g.shape[3]
    assert s.is_contiguous() and g.is_contiguous() and s.dtype == torch.bfloat16 and g.dtype == torch.bfloat16
    assert tuple(g.shape[:3]) == (B, 2 * h, 2 * w), "g must be the 2x map of s"
    out = torch.empty((M, N, 4, 4), dtype=torch.float32, device=s.device)
    ws = torch.empty(lib().cv_conv_k4s2_wgrad_workspace_bytes(B, h, w, M, N) // 4, dtype=torch.float32,
                     device=s.device)
    check(lib().cv_conv_k4s2_wgrad(ptr(s), ptr(g), ptr(out), ptr(ws), B, h, w, M, N, stream_ptr()),
          "cv_conv_k4s2_wgrad")
    return out


def relu_mask_(dx, act):
    """dx *= (act > 0) in place (ReLU backward from the saved ReLU output); both bf16, same shape."""
    require_cuda(dx, act)
    assert dx.shape == act.shape and dx.is_contiguous() and act.is_contiguous()
    assert dx.dtype == torch.bfloat16 and act.dtype == torch.bfloat16
    check(lib().cv_relu_mask_bf16(ptr(dx), ptr(act), dx.numel(), stream_ptr()), "cv_relu_mask_bf16")
    return dx


def conv1x1_out3_bwd(dr, x, w):
    """Backward of conv1x1_out3 (scale 1, shift 0) after a ReLU: dr [B, 3, H, W] fp32, x [B, H, W, Cin] bf16 (the ReLU
    output), w [3, Cin] fp32 -> (dx [B, H, W, Cin] bf16 masked by x > 0, dw [3, Cin] fp32, db [3] fp32)."""
    require_cuda(dr, x, w)
    B, H, W, Cin = x.shape
    assert dr.shape == (B, 3, H, W) and dr.dtype == torch.float32 and dr.is_contiguous()
    assert x.is_contiguous() and x.dtype == torch.bfloat16 and w.is_contiguous() and w.dtype == torch.float32
    dx = torch.empty_like(x)
    dw = torch.empty((3, Cin), dtype=torch.float32, device=x.device)
    db = torch.empty(3, dtype=torch.float32, device=x.device)
    ws = torch.empty(lib().cv_conv1x1_out3_bwd_workspace_bytes(Cin) // 4, dtype=torch.float32, device=x.device)
    check(lib().cv_conv1x1_out3_bwd(ptr(dr), ptr(x), ptr(w), ptr(dx), ptr(dw), ptr(db), ptr(ws), B, H, W, Cin,
                                    stream_ptr()), "cv_conv1x1_out3_bwd")
    return dx, dw, db


def vq_ema_stats(idx, z, n_embed):
    """idx [rows] int64 codes, z [rows, dim] fp32 -> (counts [n_embed] fp32, embed_sum [dim, n_embed] fp32)."""
    require_cuda(idx, z)
    idx = idx.contiguous().view(-1)
    rows, dim = z.shape
    assert idx.numel() == rows and idx.dtype == torch.int64 and z.dtype == torch.float32 and z.is_contiguous()
    counts = torch.empty(n_embed, dtype=torch.float32, device=z.device)
    embed_sum = torch.empty((dim, n_embed), dtype=torch.float32, device=z.device)
    check(lib().cv_vq_ema_stats(ptr(idx), ptr(z), rows, dim, n_embed, ptr(counts), ptr(embed_sum), stream_ptr()),
          "cv_vq_ema_stats")
    return counts, embed_sum


def gumbel_noise(seed, row0, rows, K, device="cuda"):
    """The Gumbel(0, 1) noise [rows, K] fp32 of absolute rows row0 .. row0 + rows - 1 that vq_gumbel_fwd / _bwd use."""
    out = torch.empty((rows, K), dtype=torch.float32, device=device)
    check(lib().cv_gumbel_noise(int(seed), int(row0), rows, K, ptr(out), stream_ptr()), "cv_gumbel_noise")
    return out


def _check_scores(scores, e2):
    require_cuda(scores, e2)
    assert scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1
    assert e2.dtype == torch.float32 and e2.is_contiguous() and e2.numel() == scores.shape[1]


def vq_gumbel_fwd(scores, e2, seed, row0, tau, *, y_dtype=torch.bfloat16, want_kl=False):
    """Gumbel softmax over the codes, per row of scores [rows, K] fp32 (z.E) and e2 [K] (|e|^2).
    Returns (y [rows, K] of y_dtype, or None when y_dtype is None; idx [rows] int64; kl [rows] fp32 or None)."""
    _check_scores(scores, e2)
    rows, K = scores.shape
    y = None if y_dtype is None else torch.empty((rows, K), dtype=y_dtype, device=scores.device)
    assert y_dtype in (None, torch.bfloat16, torch.float32)
    idx = torch.empty(rows, dtype=torch.int64, device=scores.device)
    kl = torch.empty(rows, dtype=torch.float32, device=scores.device) if want_kl else None
    check(lib().cv_vq_gumbel_fwd(ptr(scores), scores.stride(0), ptr(e2), rows, K, int(seed), int(row0), float(tau),
                                 ptr(y), int(y_dtype == torch.float32), K, ptr(idx), ptr(kl), stream_ptr()),
          "cv_vq_gumbel_fwd")
    return y, idx, kl


def vq_gumbel_bwd(scores, e2, seed, row0, tau, dy=None, kl_scale=0.0):
    """Backward of vq_gumbel_fwd's y (from dy [rows, K] fp32) and of its KL (scaled by kl_scale) to the logits
    a = 2 scores - e2.  Returns (da [rows, K] bf16, rowsum [rows] fp32 = sum_j da)."""
    _check_scores(scores, e2)
    rows, K = scores.shape
    if dy is not None:
        require_cuda(dy)
        assert dy.dtype == torch.float32 and dy.shape == (rows, K) and dy.stride(1) == 1
    da = torch.empty((rows, K), dtype=torch.bfloat16, device=scores.device)
    rowsum = torch.empty(rows, dtype=torch.float32, device=scores.device)
    check(lib().cv_vq_gumbel_bwd(ptr(scores), scores.stride(0), ptr(e2), rows, K, int(seed), int(row0), float(tau),
                                 ptr(dy), 0 if dy is None else dy.stride(0), float(kl_scale), ptr(da), K, ptr(rowsum),
                                 stream_ptr()), "cv_vq_gumbel_bwd")
    return da, rowsum


def attn_gather(q, cache, idx, heads):
    """sparse_attention_inference: q [b, sq, h] view, cache [b, max_len, 2h] (K|V), idx [b, n] int64 -> [b, sq, h]."""
    require_cuda(q, cache, idx)
    b, sq, h = q.shape
    assert q.stride(2) == 1 and cache.stride(2) == 1 and cache.stride(1) == 2 * h and idx.dtype == torch.int64
    idx = idx.contiguous()
    out = torch.empty((b, sq, h), dtype=torch.bfloat16, device=q.device)
    rc = lib().cv_attn_gather(ptr(q), q.stride(1), q.stride(0), ptr(cache), cache.stride(0), ptr(idx), ptr(out), b, heads,
                              64, sq, idx.shape[1], stream_ptr())
    check(rc, "cv_attn_gather")
    return out
