"""Test helpers for dense attention (cv_attn_fwd / cv_attn_bwd) and sparse training attention (cv_attn_sparse_fwd /
cv_attn_sparse_bwd, as dense attention over virtual keys: see the sparse section below); no GPU needed to import.

The operation is the reference's standard_attention over its two mask families, with queries the LAST sq of the sk
keys (decode-with-memory prefill when sq < sk):

    S = Q K^T / 8 on visible entries, exactly -10000 elsewhere;  P = softmax(S);  out = (P * keep / (1 - p)) V

* `visible`: the float64 mask (causal, or int `sep`: keys [0, sep + sk - sq) visible to every query), with knobs that
  move the diagonal, `sep` or `off = sk - sq` by a few keys: the off-by-one kernels the bounds must catch.
* `forward64` / `backward64`: float64 forward, lse and autograd backward on the bf16-rounded inputs.
* `fwd_bound` / `bwd_bounds`: the per-element error a bf16 kernel may legitimately make (below).
* `emulate_fwd` / `emulate_bwd`: float32/bf16 emulations of the kernels' rounding (fp32 scores and accumulators,
  online softmax over 128-key tiles, bf16 P in both the P V product and the row sum, bf16 dS and outputs).
* `keep_from_bits` / `visited_tiles`: the dropout keep bits of cv_attn_fwd decoded from both of its layouts.
* `sparse_visible` / `pivot_bias` / `virtual_keys` / `sparse_backward64` / `emulate_sparse_fwd` / `emulate_sparse_bwd`:
  the same for the sparse attention, with the knobs of its plausible bugs (window edge, diagonal, pivot test and bias,
  tile walks, pivot scatter).

Error model (u = 2^-8, the unit roundoff of bf16's 8 significant bits):
  forward   |out - ref| <= 2u |ref| + u (P |V|) + 1e-5       (bf16 P in numerator and row sum, bf16 output)
  lse       |lse - ref| <= 2u + 1e-5
  backward  |g - ref| <= u |ref| + c u X + 1e-5,  with X the same product taken on absolute values:
            dV: P^T |dO|;  dQ: scale (P o (|dP| + |D| + dD)) |K|;  dK: scale (P o (|dP| + |D| + dD))^T |Q|
            dP = dO V^T (through the keep mask), D = rowsum(dO o O), dD = sum_d |dO| (2 |O| + P |V|), the forward
            bound in units of u: the kernel builds D from its own bf16 O, so D is off by up to u dD, and that error
            enters dS unscaled by the u of the term it sits in.  With dropout, dV's P and dP carry keep / (1 - p); dS keeps the undropped P.
C_BWD is the smallest integer for which the emulated backward stays within 0.75 of this bound
(tests/test_attention_bounds_cpu.py).
"""
import math

import torch

U = 2.0 ** -8
FLOOR = 1e-5
C_BWD = 2
T = 128                     # keys per tile and queries per block of both kernels
HD = 64
SCALE = 1.0 / math.sqrt(HD)
LOG2E = 1.4426950408889634
MASKED = -10000.0


# ----------------------------------------------------------------------------------------------------
# masks
# ----------------------------------------------------------------------------------------------------
def visible(sq, sk, sep, *, diag=0, sep_shift=0, off_shift=0, device=None):
    """[sq, sk] bool: key j visible to query i.  Query i is sequence position i + off (off = sk - sq); it sees the
    keys j <= i + off (causal) and the keys j < sep + off (the reference marks [0, sep + mem) visible, also for
    sep = 0, where those keys are causally visible anyway).  diag / sep_shift / off_shift move the causal diagonal,
    `sep`, or `off` in both places, by that many keys."""
    off = sk - sq + off_shift
    i = torch.arange(sq, device=device)[:, None]
    j = torch.arange(sk, device=device)[None, :]
    return (j <= i + off + diag) | (j < sep + sep_shift + off)


def visited_tiles(sq, sk, sep, device=None):
    """[sq, sk] bool: (query, key) pairs inside the key tiles the forward visits for the query's 128-query block:
    tiles below max(q0 + 128 + off, sep + off), the tiles whose dropout keep bits are written."""
    off = sk - sq
    qb = torch.arange(sq, device=device) // T
    kmax = torch.clamp(torch.maximum(qb * T + T + off, torch.full_like(qb, sep + off if sep > 0 else 0)), max=sk)
    ntiles = (kmax + T - 1) // T
    return (torch.arange(sk, device=device)[None, :] // T) < ntiles[:, None]


def heads_of(t, heads):
    """[b, s, heads*64] -> [b, heads, s, 64]."""
    b, s, _ = t.shape
    return t.reshape(b, s, heads, HD).permute(0, 2, 1, 3)


# ----------------------------------------------------------------------------------------------------
# float64 reference and bounds
# ----------------------------------------------------------------------------------------------------
def _keep_scale(keep, p):
    return None if keep is None else keep.double() / (1.0 - p)


def forward64(q, k, v, vis, keep=None, p=0.0, bias=None):
    """q [..., sq, 64], k / v [..., sk, 64] (any float dtype; computed in float64), vis [sq, sk], keep [..., sq, sk]
    0/1 or None, bias [sk] float64 or None: added to the visible scores of each key (the sparse pivot bias).
    Returns out, lse (natural log, of the undropped scores) and the undropped probabilities P."""
    q, k, v = q.double(), k.double(), v.double()
    x = (q @ k.transpose(-1, -2)) * SCALE
    if bias is not None:
        x = x + bias
    s = torch.where(vis, x, torch.full((), MASKED, dtype=torch.float64, device=q.device))
    lse = torch.logsumexp(s, dim=-1)
    probs = torch.exp(s - lse[..., None])
    ks = _keep_scale(keep, p)
    return (probs if ks is None else probs * ks) @ v, lse, probs


def fwd_bound(out, probs, v, keep=None, p=0.0):
    """Per-element bound of |out_kernel - out| (out, probs from forward64)."""
    ks = _keep_scale(keep, p)
    return 2 * U * out.abs() + U * ((probs if ks is None else probs * ks) @ v.double().abs()) + FLOOR


def lse_bound():
    return 2 * U + FLOOR


def backward64(q, k, v, d_out, vis, keep=None, p=0.0, bias=None):
    """Float64 autograd of forward64.  Returns (dq, dk, dv), out and the undropped probabilities."""
    q, k, v = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    out, _, probs = forward64(q, k, v, vis, keep, p, bias)
    out.backward(d_out.double())
    return (q.grad, k.grad, v.grad), out.detach(), probs.detach()


def bwd_bounds(q, k, v, d_out, out, probs, grads, keep=None, p=0.0, c=C_BWD):
    """Per-element bounds of the dq, dk, dv errors (out, probs, grads from backward64)."""
    q, k, v, d_out = q.double(), k.double(), v.double(), d_out.double()
    dq, dk, dv = grads
    ks = _keep_scale(keep, p)
    dp = d_out @ v.transpose(-1, -2)
    pdrop = probs
    if ks is not None:
        dp = dp * ks
        pdrop = probs * ks
    d = (d_out * out).sum(-1, keepdim=True)
    dd = (d_out.abs() * (2 * out.abs() + pdrop @ v.abs())).sum(-1, keepdim=True)   # dD / u
    g = probs * (dp.abs() + d.abs() + dd)                  # |dS| / scale, term by term
    bq = U * dq.abs() + c * U * SCALE * (g @ k.abs()) + FLOOR
    bk = U * dk.abs() + c * U * SCALE * (g.transpose(-1, -2) @ q.abs()) + FLOOR
    bv = U * dv.abs() + c * U * (pdrop.transpose(-1, -2) @ d_out.abs()) + FLOOR
    return bq, bk, bv


def ratio(got, ref, bound):
    """Worst |got - ref| / bound (NaN or inf in got counts as infinitely far)."""
    err = (got.double() - ref).abs() / bound
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, math.inf))
    return err.max().item() if err.numel() else 0.0


# ----------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------
def make_inputs(b, heads, sq, sk, std, order, generator, device="cpu", pivots=None):
    """bf16 q [b, sq, heads*64], k / v [b, sk, heads*64] whose scores Q K^T / 8 have standard deviation `std`.
    order 'random': i.i.d.; 'rising': each later key tile adds 6 std to every score, so the running maximum of the
    online softmax rises in every tile; 'first': the first key tile carries +6 std, so the maximum sits there;
    'pivot': the keys at the positions pivots [b, n_piv] carry +6 std, so a query that sees pivots takes most of its
    weight from them."""
    sigma = math.sqrt(std)
    q = torch.randn((b, sq, heads, HD), generator=generator, device=device) * sigma
    k = torch.randn((b, sk, heads, HD), generator=generator, device=device) * sigma
    v = torch.randn((b, sk, heads, HD), generator=generator, device=device)
    if order == "pivot":
        mark = torch.zeros((b, sk), device=device)
        mark.scatter_(1, pivots.to(device), 1.0)
        q[..., 0] = 8.0
        k[..., 0] = (mark * 6.0 * std)[:, :, None]
    elif order != "random":
        tile = torch.arange(sk, device=device) // T
        step = (tile.float() if order == "rising" else (tile == 0).float()) * 6.0 * std
        q[..., 0] = 8.0                                  # score bias = q0 * k0 / 8 = k0
        k[..., 0] = step[None, :, None]
    return tuple(t.reshape(t.shape[0], t.shape[1], heads * HD).to(torch.bfloat16) for t in (q, k, v))


# ----------------------------------------------------------------------------------------------------
# float32 / bf16 emulations of the kernels' rounding
# ----------------------------------------------------------------------------------------------------
def _bf(x):
    return x.to(torch.bfloat16).float()


SCALE_LOG2 = torch.tensor(SCALE * LOG2E, dtype=torch.float32).item()
MASKED_LOG2 = torch.tensor(MASKED * LOG2E, dtype=torch.float32).item()


def emulate_fwd(q, k, v, vis, keep=None, p=0.0, *, drop_tile=None, drop_scale_power=1):
    """cv_attn_fwd in float32 / bf16 on [..., s, 64] inputs: for each 128-query block, the key tiles up to the last
    key any of its queries sees, fp32 scores in the log2 domain, online softmax, P rounded to bf16 for both the P V
    product and the row sum, dropout on the bf16 P with the 1/(1-p) scale applied once to the output row, bf16 output.
    Mutations: drop_tile = (query block, key tile) skips that tile for that block; drop_scale_power = 2 applies the
    dropout scale twice.  Returns out (bf16 values, float32) and lse (float32)."""
    sq, sk = q.shape[-2], k.shape[-2]
    tiles = []
    for qb in range((sq + T - 1) // T):
        kmax = int(vis[qb * T:qb * T + T].nonzero()[:, 1].max().item()) + 1
        tiles.append([slice(j * T, min(sk, j * T + T)) for j in range((kmax + T - 1) // T) if drop_tile != (qb, j)])
    return _emulate_fwd_tiles(q, k, v, vis, tiles, keep, p, None, drop_scale_power)


def _emulate_fwd_tiles(q, k, v, vis, tiles, keep, p, bias, drop_scale_power):
    """The forward kernel's online softmax: query block qb walks the key column ranges tiles[qb] in order; bias [sk]
    (float64 or None) is added to the visible scores in the log2 domain, in float32."""
    q, k, v = q.float(), k.float(), v.float()
    sq = q.shape[-2]
    bias2 = None if bias is None else (bias * LOG2E).float()
    scale = (1.0 / (1.0 - p)) ** drop_scale_power if keep is not None else 1.0
    outs, lses = [], []
    for qb in range((sq + T - 1) // T):
        rows = slice(qb * T, min(sq, qb * T + T))
        vr = vis[rows]
        m = torch.full(q[..., rows, 0].shape, -math.inf)
        l = torch.zeros_like(m)
        o = torch.zeros(q[..., rows, :].shape)
        for ks in tiles[qb]:
            x = (q[..., rows, :] @ k[..., ks, :].transpose(-1, -2)) * SCALE_LOG2
            if bias2 is not None:
                x = x + bias2[ks]
            x = torch.where(vr[:, ks], x, torch.full((), MASKED_LOG2))
            mx = torch.maximum(m, x.amax(-1))
            alpha = torch.exp2(m - mx)
            m = mx
            pe = _bf(torch.exp2(x - m[..., None]))
            l = l * alpha + pe.sum(-1)
            if keep is not None:
                pe = pe * keep[..., rows, ks].float()
            o = o * alpha[..., None] + pe @ v[..., ks, :]
        outs.append(_bf(o * (scale / l)[..., None]))
        lses.append(m * math.log(2.0) + torch.log(l))
    return torch.cat(outs, -2), torch.cat(lses, -1)


def emulate_bwd(q, k, v, out, d_out, lse, vis, keep=None, p=0.0, *, drop_tile=None, drop_scale_power=1):
    """cv_attn_bwd in float32 / bf16 (sq == sk), given the (emulated) kernel forward's bf16 out and fp32 lse: P
    recomputed from lse in the log2 domain, D = rowsum(dO o O) from the bf16 O, dS = P o (dP - D) * scale in fp32,
    P (dropped) and dS rounded to bf16 for the three products, fp32 accumulation, bf16 outputs.  Mutations:
    drop_tile = (query block, key block) leaves that tile out; drop_scale_power = 2 applies the dropout scale twice."""
    q, k, v, out, d_out = (t.float() for t in (q, k, v, out, d_out))
    s = q.shape[-2]
    x = torch.where(vis, (q @ k.transpose(-1, -2)) * SCALE_LOG2, torch.full((), MASKED_LOG2))
    prob = torch.exp2(x - (lse.float() * LOG2E)[..., None])
    if drop_tile is not None:
        qb, kb = drop_tile
        prob = prob.clone()
        prob[..., qb * T:min(s, qb * T + T), kb * T:min(s, kb * T + T)] = 0.0
    dp = d_out @ v.transpose(-1, -2)
    d = (d_out * out).sum(-1, keepdim=True)
    pdrop = prob
    if keep is not None:
        ks = keep.float() * (1.0 / (1.0 - p)) ** drop_scale_power
        dp = dp * ks
        pdrop = prob * ks
    ds = prob * (dp - d) * SCALE
    dsb = _bf(ds)
    dv = _bf(_bf(pdrop).transpose(-1, -2) @ d_out)
    dk = _bf(dsb.transpose(-1, -2) @ q)
    dq = _bf(dsb @ k)
    return dq, dk, dv


# ----------------------------------------------------------------------------------------------------
# sparse training attention (cv_attn_sparse_fwd / cv_attn_sparse_bwd) as dense attention over virtual keys
# ----------------------------------------------------------------------------------------------------
# The sparse attention of one batch row is an ordinary softmax over s + n_piv VIRTUAL keys: the s sequence keys
# (band), then the n_piv gathered pivot keys K[pivots], V[pivots] (slots), with
#     band  j:  band_start(i) <= j <= i,        band_start(i) = max(0, i // w - times + 1) * w
#     slot  p:  pivots[p] < band_start(i),      score + log(s // n_piv)
# (tests/test_attention_sparse_bounds_cpu.py proves it equal to the oracle's sparse_attention).  So forward64, fwd_bound
# and backward64 apply unchanged to the virtual keys; the bounds need no bias (they are functions of P alone).
def band_start(i, w, times):
    return torch.clamp(i // w - times + 1, min=0) * w


def sparse_visible(s, w, times, pivots, *, band_shift=0, times_shift=0, diag=0, piv_le=False):
    """[s, s + n_piv] bool over the virtual keys of one batch row (pivots [n_piv]).  Mutations: band_shift moves the
    band's first key by that many keys (for queries whose band does not start at 0); times_shift changes `times` in
    band_start (band and pivot test); diag moves the causal diagonal; piv_le tests pivots[p] <= band_start(i)."""
    dev = pivots.device
    i = torch.arange(s, device=dev)[:, None]
    j = torch.arange(s, device=dev)[None, :]
    bs = band_start(i, w, times + times_shift)
    band = (j >= torch.where(bs > 0, bs + band_shift, bs)) & (j <= i + diag)
    pos = pivots[None, :]
    piv = (pos <= bs) if piv_le else (pos < bs)
    return torch.cat((band, piv), dim=1)


def pivot_bias(s, n_piv, mode="floor", device=None):
    """[s + n_piv] float64: 0 on the band keys, log(s // n_piv) on the pivot slots ('floor', the reference); mutations
    'none' (no bias) and 'div' (log(s / n_piv))."""
    b = torch.zeros(s + n_piv, dtype=torch.float64, device=device)
    if mode != "none":
        b[s:] = math.log(s // n_piv) if mode == "floor" else math.log(s / n_piv)
    return b


def virtual_keys(k, pivots):
    """[..., s, 64] -> [..., s + n_piv, 64]: the sequence keys, then the gathered pivot keys."""
    return torch.cat((k, k[..., pivots, :]), dim=-2)


def sparse_backward64(q, k, v, d_out, pivots, vis, bias, keep=None, p=0.0, c=C_BWD):
    """Float64 gradients and bounds of the sparse attention of one batch row.  The autograd runs over the virtual keys;
    dK / dV of a sequence position = its band part + the part of the pivot slot that gathers it.  The kernel rounds
    the two parts to bf16 separately and their sum once more, so a pivot position's bound is the band bound + the
    slot bound + u (|band part| + |slot part|).  dQ accumulates both passes in fp32 and keeps the dense bound.
    Returns (dq, dk, dv), (bq, bk, bv)."""
    s = k.shape[-2]
    kv, vv = virtual_keys(k, pivots), virtual_keys(v, pivots)
    (dq, dkv, dvv), out, probs = backward64(q, kv, vv, d_out, vis, keep, p, bias)
    bq, bkv, bvv = bwd_bounds(q, kv, vv, d_out, out, probs, (dq, dkv, dvv), keep, p, c)
    is_piv = torch.zeros(s, dtype=torch.float64, device=q.device)
    is_piv[pivots] = 1.0

    def fold(g):
        return g[..., :s, :].index_add(-2, pivots, g[..., s:, :])

    def fold_bound(bd, g):
        extra = U * g[..., :s, :].abs() * is_piv[:, None]
        return (bd[..., :s, :] + extra).index_add(-2, pivots, bd[..., s:, :] + U * g[..., s:, :].abs())
    return (dq, fold(dkv), fold(dvv)), (bq, fold_bound(bkv, dkv), fold_bound(bvv, dvv))


def sparse_walk(s, w, times):
    """The tile walks of csrc/attention_sparse.cuh: per query block, the forward's band key tiles and whether it
    visits the pivot tiles; per key block, the last query block of the backward band pass; the first query block of
    the pivot pass (None: the pivot pass is not launched)."""
    nqb = (s + T - 1) // T
    last = [min(qb * T + T, s) - 1 for qb in range(nqb)]
    first = [int(band_start(torch.tensor(qb * T), w, times)) // T for qb in range(nqb)]
    band = [list(range(first[qb], last[qb] // T + 1)) for qb in range(nqb)]
    sees = [int(band_start(torch.tensor(last[qb]), w, times)) > 0 for qb in range(nqb)]
    band_last = [min(nqb - 1, (((kb * T + T - 1) // w + times) * w - 1) // T) for kb in range(nqb)]
    piv_first = (times * w) // T if times * w < s else None
    return dict(band=band, sees=sees, band_last=band_last, piv_first=piv_first)


def emulate_sparse_fwd(q, k, v, pivots, w, times, vis, bias, keep=None, p=0.0, *, drop_tile=None,
                       sees_pivots_first_query=False, drop_scale_power=1):
    """cv_attn_sparse_fwd in float32 / bf16 for one batch row: query block qb walks its band key tiles, then every
    pivot tile if its last query sees pivots, as one online softmax over the virtual keys (emulate_fwd).  Mutations:
    drop_tile = (qb, 'band', j) skips the j-th band tile of the block's walk, (qb, 'piv', t) pivot tile t;
    sees_pivots_first_query decides the pivot tiles from the block's FIRST query; drop_scale_power = 2."""
    s, n_piv = k.shape[-2], pivots.shape[0]
    walk = sparse_walk(s, w, times)
    tiles = []
    for qb in range((s + T - 1) // T):
        ts = [slice(jb * T, min(s, jb * T + T)) for j, jb in enumerate(walk["band"][qb]) if drop_tile != (qb, "band", j)]
        sees = walk["sees"][qb]
        if sees_pivots_first_query:
            sees = int(band_start(torch.tensor(qb * T), w, times)) > 0
        if sees:
            ts += [slice(s + t * T, s + min(n_piv, t * T + T)) for t in range((n_piv + T - 1) // T)
                   if drop_tile != (qb, "piv", t)]
        tiles.append(ts)
    return _emulate_fwd_tiles(q, virtual_keys(k, pivots), virtual_keys(v, pivots), vis, tiles, keep, p, bias,
                              drop_scale_power)


def emulate_sparse_bwd(q, k, v, pivots, w, times, out, d_out, lse, vis, bias, keep=None, p=0.0, *, band_last_shift=0,
                       piv_first_shift=0, scatter="once", drop_scale_power=1):
    """cv_attn_sparse_bwd in float32 / bf16 for one batch row, given the kernel forward's bf16 out and fp32 lse: the
    band pass (key block kb, query blocks kb .. band_last(kb)) and the pivot pass (query blocks piv_first ..) over the
    virtual keys as emulate_bwd, P from the joint lse (bias added in the log2 domain), D from the bf16 O; dQ of both
    passes in fp32, rounded once; the band and pivot-slot dK / dV each rounded to bf16, and the slot part then added
    onto its position and rounded again.  Mutations: band_last_shift / piv_first_shift move the walk bounds;
    scatter 'skip', 'twice' or 'next' (onto position + 1); drop_scale_power = 2."""
    q, out, d_out = q.float(), out.float(), d_out.float()
    s, n_piv = k.shape[-2], pivots.shape[0]
    kv, vv = virtual_keys(k.float(), pivots), virtual_keys(v.float(), pivots)
    walk = sparse_walk(s, w, times)
    covered = torch.zeros((s, s + n_piv), dtype=torch.bool)
    for kb, last in enumerate(walk["band_last"]):
        covered[kb * T:(last + band_last_shift) * T + T, kb * T:kb * T + T] = True
    if walk["piv_first"] is not None:
        covered[(walk["piv_first"] + piv_first_shift) * T:, s:] = True
    x = (q @ kv.transpose(-1, -2)) * SCALE_LOG2 + (bias * LOG2E).float()
    x = torch.where(vis, x, torch.full((), MASKED_LOG2))
    prob = torch.exp2(x - (lse.float() * LOG2E)[..., None]) * covered
    dp = d_out @ vv.transpose(-1, -2)
    d = (d_out * out).sum(-1, keepdim=True)
    pdrop = prob
    if keep is not None:
        ks = keep.float() * (1.0 / (1.0 - p)) ** drop_scale_power
        dp = dp * ks
        pdrop = prob * ks
    dsb = _bf(prob * (dp - d) * SCALE)
    dq = _bf(dsb @ kv)
    grads = []
    for g in (dsb.transpose(-1, -2) @ q, _bf(pdrop).transpose(-1, -2) @ d_out):
        band, slot = _bf(g[..., :s, :]), _bf(g[..., s:, :])
        if walk["piv_first"] is not None and scatter != "skip":
            dst = (pivots + 1) % s if scatter == "next" else pivots
            for _ in range(2 if scatter == "twice" else 1):
                band[..., dst, :] = _bf(band[..., dst, :] + slot)
        grads.append(band)
    return dq, grads[0], grads[1]


# ----------------------------------------------------------------------------------------------------
# dropout keep bits
# ----------------------------------------------------------------------------------------------------
def keep_from_bits(mask, sq, sk):
    """mask: the int32 keep-bit buffer of cv_attn_fwd, [2, b, heads, ceil(sk/128)*ceil(sq/128)*128, 4].
    [0] key-major [b, heads, key (padded), query block, 4] words, bit i of word w = query qb*128 + 32w + i;
    [1] query-major [b, heads, query (padded), key block, 4].  Returns keep [b, heads, sq, sk] from each layout."""
    _, b, heads, _, _ = mask.shape
    nkb, nqb = (sk + T - 1) // T, (sq + T - 1) // T
    words = mask.to(torch.int64) & 0xFFFFFFFF
    sh = torch.arange(32, device=mask.device)
    kmaj = ((words[0].view(b, heads, nkb * T, nqb, 4).unsqueeze(-1) >> sh) & 1).reshape(b, heads, nkb * T, nqb * T)
    qmaj = ((words[1].view(b, heads, nqb * T, nkb, 4).unsqueeze(-1) >> sh) & 1).reshape(b, heads, nqb * T, nkb * T)
    return kmaj[:, :, :sk, :sq].transpose(2, 3), qmaj[:, :, :sq, :sk]
