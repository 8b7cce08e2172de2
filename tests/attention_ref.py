"""Test helpers for dense attention (cv_attn_fwd / cv_attn_bwd); no GPU needed to import.

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


def forward64(q, k, v, vis, keep=None, p=0.0):
    """q [..., sq, 64], k / v [..., sk, 64] (any float dtype; computed in float64), vis [sq, sk], keep [..., sq, sk]
    0/1 or None.  Returns out, lse (natural log, of the undropped scores) and the undropped probabilities P."""
    q, k, v = q.double(), k.double(), v.double()
    s = torch.where(vis, (q @ k.transpose(-1, -2)) * SCALE, torch.full((), MASKED, dtype=torch.float64,
                                                                     device=q.device))
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


def backward64(q, k, v, d_out, vis, keep=None, p=0.0):
    """Float64 autograd of forward64.  Returns (dq, dk, dv), out and the undropped probabilities."""
    q, k, v = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    out, _, probs = forward64(q, k, v, vis, keep, p)
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
def make_inputs(b, heads, sq, sk, std, order, generator, device="cpu"):
    """bf16 q [b, sq, heads*64], k / v [b, sk, heads*64] whose scores Q K^T / 8 have standard deviation `std`.
    order 'random': i.i.d.; 'rising': each later key tile adds 6 std to every score, so the running maximum of the
    online softmax rises in every tile; 'first': the first key tile carries +6 std, so the maximum sits there."""
    sigma = math.sqrt(std)
    q = torch.randn((b, sq, heads, HD), generator=generator, device=device) * sigma
    k = torch.randn((b, sk, heads, HD), generator=generator, device=device) * sigma
    v = torch.randn((b, sk, heads, HD), generator=generator, device=device)
    if order != "random":
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
    q, k, v = q.float(), k.float(), v.float()
    sq, sk = q.shape[-2], k.shape[-2]
    scale = (1.0 / (1.0 - p)) ** drop_scale_power if keep is not None else 1.0
    outs, lses = [], []
    for qb in range((sq + T - 1) // T):
        rows = slice(qb * T, min(sq, qb * T + T))
        vr = vis[rows]
        kmax = int(vr.nonzero()[:, 1].max().item()) + 1
        m = torch.full(q[..., rows, 0].shape, -math.inf)
        l = torch.zeros_like(m)
        o = torch.zeros(q[..., rows, :].shape)
        for j in range((kmax + T - 1) // T):
            if drop_tile == (qb, j):
                continue
            ks = slice(j * T, min(sk, j * T + T))
            x = (q[..., rows, :] @ k[..., ks, :].transpose(-1, -2)) * SCALE_LOG2
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
