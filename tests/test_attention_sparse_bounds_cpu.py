"""The per-element error bounds of sparse training attention are the yardstick of tests/test_attention_sparse_gpu.py.
These CPU tests are the argument that the yardstick is right:

* the float64 reference of tests/attention_ref.py, one softmax over the VIRTUAL keys (the s sequence keys, then the
  n_piv gathered pivot keys, visible as band_start(i) <= j <= i and pivots[p] < band_start(i), + log(s // n_piv) on
  the pivot slots), equals the oracle's sparse_attention in float64, with and without dropout, values and gradients;
* an emulation of the two kernels' rounding and tile walks (attention_ref.emulate_sparse_fwd / _bwd) stays within 0.75
  of every bound, at both score scales and every key ordering, with and without dropout;
* the same emulation with one plausible kernel bug (a window edge, the diagonal, the pivot test or bias, a tile of the
  walk, the pivot scatter, the dropout scale or a keep bit) exceeds the bound on the case named beside it, at score
  std 1 and 6, so a kernel with that bug would fail the GPU test.

The backward bound uses the dense constant c = 2 (attention_ref.C_BWD); with c = 1 the emulated dV reaches 0.95 of
its bound on these cases, so 2 is again the smallest integer that keeps every backward ratio within 0.75.  The dropout
forward is held to the dense test's 0.85: the same cancellation (a row whose largest probability is dropped, leaving
kept terms of opposite sign rounded the same way) applies unchanged, since the virtual keys are an ordinary softmax.
"""
import math

import pytest
import torch

import attention_ref as R
import sparse_dropout_ref as SD
from oracle import cogview_oracle as O
from oracle import sparse_decomposition as SDEC

P_DROP = 0.1
STDS = (1.0, 6.0)
ORDERS = ("random", "rising", "first", "pivot")


def planted_pivots(s, w, times):
    """Pivot positions on both sides of every window edge's band start (band_start(i) - 1 and band_start(i) for the
    window-edge queries i = g*w and g*w - 1), and the tile edges 0, 127, 128, s - 1."""
    pos = {0, 127, 128, s - 1}
    for g in range(1, s // w + 1):
        for i in (g * w, g * w - 1):
            if i < s:
                bs = int(R.band_start(torch.tensor(i), w, times))
                pos |= {bs - 1, bs} if bs > 0 else set()
    return torch.tensor(sorted(x for x in pos if 0 <= x < s), dtype=torch.long)


def make_pivots(kind, s, n_piv, generator):
    """'ref': the reference's order (text positions first, then a random sample of the rest); 'desc': a random set in
    descending order (the last slot holds the smallest position); 'planted': planted_pivots."""
    if kind == "planted":
        raise ValueError("planted pivots depend on w and times")
    txt = min(n_piv // 3, 20)
    rest = txt + torch.randperm(s - txt, generator=generator)[:n_piv - txt]
    piv = torch.cat((torch.arange(txt), rest))
    return piv.sort(descending=True).values if kind == "desc" else piv


def _inputs(s, w, times, n_piv, heads, std, order, pivot_kind="ref", seed=0):
    """One batch row in heads-first layout: q, k, v [1, heads, s, 64] bf16, pivots [n_piv], keep [1, heads, s, s+n_piv]
    (0/1 over the virtual keys), d_out."""
    g = torch.Generator().manual_seed(7919 * s + 31 * w + times + 3 * (n_piv or 0) + int(std) + seed)
    pivots = planted_pivots(s, w, times) if pivot_kind == "planted" else make_pivots(pivot_kind, s, n_piv, g)
    q, k, v = (R.heads_of(t, heads) for t in R.make_inputs(1, heads, s, s, std, order, g, pivots=pivots[None]))
    keep = torch.rand((1, heads, s, s + pivots.shape[0]), generator=g) >= P_DROP
    d_out = torch.randn((1, heads, s, 64), generator=g).to(torch.bfloat16)
    return q, k, v, pivots, keep, d_out


# ----------------------------------------------------------------------------------------------------
# the virtual-key reference is the oracle's sparse attention
# ----------------------------------------------------------------------------------------------------
def _rmask(s, w, times):
    g = s // w
    tmp = torch.tril(1 - torch.block_diag(*torch.ones((g - times + 1, w, w), dtype=torch.float64)))
    return torch.nn.functional.pad(tmp, (0, (times - 1) * w, (times - 1) * w, 0))


# (s, w, times, n_piv): s // n_piv with a remainder and a partial pivot tile; n_piv = s with w = 96; s = times * w (no
# query sees a pivot); a long band; s < times * w
EQUIV_CASES = [(320, 64, 3, 129), (576, 96, 2, 576), (384, 128, 3, 40), (1024, 128, 2, 300), (640, 128, 6, 40)]


@pytest.mark.parametrize("s,w,times,n_piv", EQUIV_CASES)
def test_virtual_key_reference_equals_the_oracle(s, w, times, n_piv):
    b, heads = 2, 2
    g = torch.Generator().manual_seed(s + n_piv)
    q, k, v = (torch.randn((b, heads, s, 64), generator=g, dtype=torch.float64) * 2 for _ in range(3))
    pivots = torch.stack([make_pivots("ref", s, n_piv, g) for _ in range(b)])
    band, piv = SDEC.visibility(s, pivots, w, times)
    pam = piv.double()                          # the pivot mask in closed form
    if s >= times * w:                          # the reference's rmask cannot be built for s < times * w
        rpam = _rmask(s, w, times).expand(b, s, s).gather(-1, pivots.unsqueeze(1).expand(b, s, n_piv))
        assert torch.equal(rpam, pam)
    nkb, npb = (s + 127) // 128, (n_piv + 127) // 128
    keep_v = (torch.rand((b, heads, s, (nkb + npb) * 128), generator=g) >= P_DROP).to(torch.int8)
    keep_ref = SD.to_reference_layout(keep_v, s, n_piv, w, times)
    d_out = torch.randn((b, heads, s, 64), generator=g, dtype=torch.float64)
    for dropout in (False, True):
        leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
        if dropout:
            ref = SD.sparse_attention_keep(*leaves, pivots, pam, w, times, keep=keep_ref, dropout_p=P_DROP)
        else:
            ref = O.sparse_attention(*leaves, pivots, pam, w, times)
        ref.backward(d_out)
        for bi in range(b):
            vis = R.sparse_visible(s, w, times, pivots[bi])
            assert torch.equal(vis[:, :s], band) and torch.equal(vis[:, s:], piv[bi])
            kp = torch.cat((keep_v[bi:bi + 1, ..., :s], keep_v[bi:bi + 1, ..., nkb * 128:nkb * 128 + n_piv]), -1) \
                if dropout else None
            p = P_DROP if dropout else 0.0
            bias = R.pivot_bias(s, n_piv)
            out, _, _ = R.forward64(q[bi:bi + 1], R.virtual_keys(k[bi:bi + 1], pivots[bi]),
                                    R.virtual_keys(v[bi:bi + 1], pivots[bi]), vis, kp, p, bias)
            assert (out - ref[bi:bi + 1]).abs().max().item() < 1e-12
            grads, _ = R.sparse_backward64(q[bi:bi + 1], k[bi:bi + 1], v[bi:bi + 1], d_out[bi:bi + 1], pivots[bi], vis,
                                           bias, kp, p)
            for got, leaf in zip(grads, leaves):
                assert (got - leaf.grad[bi:bi + 1]).abs().max().item() < 1e-10


def test_pivot_bias_is_built_in_float64():
    """A float32 log 2 alone is off by 5e-9: the bias is computed in float64."""
    assert R.pivot_bias(320, 129)[-1].item() == math.log(2)
    assert R.pivot_bias(320, 129).dtype == torch.float64


# ----------------------------------------------------------------------------------------------------
# emulated kernels against the bounds
# ----------------------------------------------------------------------------------------------------
def _fwd_ratios(q, k, v, pivots, w, times, keep, p, *, vis_mut=None, bias_mode="floor", keep_slot_from_band=False,
                **emu):
    s, n_piv = k.shape[-2], pivots.shape[0]
    vis = R.sparse_visible(s, w, times, pivots)
    ekeep = keep
    if keep_slot_from_band:
        ekeep = keep.clone()
        ekeep[..., s:] = keep[..., :n_piv]
    out, lse = R.emulate_sparse_fwd(q, k, v, pivots, w, times, R.sparse_visible(s, w, times, pivots, **(vis_mut or {})),
                                    R.pivot_bias(s, n_piv, bias_mode), ekeep, p, **emu)
    ref, lse_ref, probs = R.forward64(q, R.virtual_keys(k, pivots), R.virtual_keys(v, pivots), vis, keep, p,
                                      R.pivot_bias(s, n_piv))
    return (R.ratio(out, ref, R.fwd_bound(ref, probs, R.virtual_keys(v, pivots), keep, p)),
            R.ratio(lse, lse_ref, R.lse_bound()))


def _bwd_ratios(q, k, v, d_out, pivots, w, times, keep, p, *, vis_mut=None, bias_mode="floor", c=R.C_BWD, **emu):
    """Worst (dq, dk, dv) ratios of the emulated backward (mutated as asked; the forward it is given is correct)."""
    s, n_piv = k.shape[-2], pivots.shape[0]
    vis, bias = R.sparse_visible(s, w, times, pivots), R.pivot_bias(s, n_piv)
    out, lse = R.emulate_sparse_fwd(q, k, v, pivots, w, times, vis, bias, keep, p)
    got = R.emulate_sparse_bwd(q, k, v, pivots, w, times, out, d_out, lse,
                               R.sparse_visible(s, w, times, pivots, **(vis_mut or {})),
                               R.pivot_bias(s, n_piv, bias_mode), keep, p, **emu)
    grads, bounds = R.sparse_backward64(q, k, v, d_out, pivots, vis, bias, keep, p, c)
    return tuple(R.ratio(gt, gr, bd) for gt, gr, bd in zip(got, grads, bounds))


# (s, w, times, n_piv, heads, pivot kind): a partial pivot tile and a block straddling times * w; n_piv = s with
# w = 96; s = times * w (no pivot pass); a small window with pivots planted at every band edge
CASES = [(320, 64, 3, 129, 2, "ref"), (576, 96, 2, 576, 1, "ref"), (384, 128, 3, 40, 1, "ref"),
         (256, 16, 4, None, 2, "planted")]


@pytest.mark.parametrize("s,w,times,n_piv,heads,kind", CASES)
def test_emulated_kernels_stay_within_the_bounds(s, w, times, n_piv, heads, kind):
    worst = {}
    for std in STDS:
        for order in ORDERS:
            for dropout in (False, True):
                q, k, v, pivots, keep, d_out = _inputs(s, w, times, n_piv, heads, std, order, kind)
                kp, p = (keep, P_DROP) if dropout else (None, 0.0)
                tag = "drop" if dropout else "nodrop"
                fo, fl = _fwd_ratios(q, k, v, pivots, w, times, kp, p)
                worst["out_" + tag] = max(worst.get("out_" + tag, 0.0), fo)
                worst["lse"] = max(worst.get("lse", 0.0), fl)
                for name, r in zip(("dq", "dk", "dv"), _bwd_ratios(q, k, v, d_out, pivots, w, times, kp, p)):
                    worst[name] = max(worst.get(name, 0.0), r)
                for name, r in zip(("dq", "dk", "dv"), _bwd_ratios(q, k, v, d_out, pivots, w, times, kp, p, c=1)):
                    worst[name + "_c1"] = max(worst.get(name + "_c1", 0.0), r)
    print("emulation / bound, worst over score std %s and orders %s:" % (STDS, ORDERS),
          " ".join("%s %.3f" % kv for kv in sorted(worst.items())))
    limits = {"out_drop": 0.85}
    for name, r in worst.items():
        if not name.endswith("_c1"):
            assert r <= limits.get(name, 0.75), (name, r)


def test_backward_constant_is_the_smallest_that_keeps_within_075():
    """With c = 1 some backward ratio passes 0.75 (so c = 2 is the smallest integer constant that does not)."""
    worst = 0.0
    for std in STDS:
        for order in ORDERS:
            q, k, v, pivots, keep, d_out = _inputs(320, 64, 3, 129, 2, std, order)
            for kp, p in ((None, 0.0), (keep, P_DROP)):
                worst = max(worst, max(_bwd_ratios(q, k, v, d_out, pivots, 64, 3, kp, p, c=1)))
    print("backward with c = 1: worst emulation / bound %.3f" % worst)
    assert worst > 0.75


# ----------------------------------------------------------------------------------------------------
# mutations: each must push the emulation past the bound at both score scales
# ----------------------------------------------------------------------------------------------------
# (name, (s, w, times, n_piv, heads, pivot kind), order, dropout, forward mutation)
FWD_MUTATIONS = [
    ("band start +1 at window edges", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(band_shift=1))),
    ("band start -1 at window edges", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(band_shift=-1))),
    ("times +1", (320, 64, 3, 129, 2, "ref"), "random", False, dict(vis_mut=dict(times_shift=1))),
    ("times -1", (320, 64, 3, 129, 2, "ref"), "random", False, dict(vis_mut=dict(times_shift=-1))),
    ("diagonal +1", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(diag=1))),
    ("diagonal -1", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(diag=-1))),
    ("pivot test <= with pivots planted at band starts", (256, 16, 2, None, 2, "planted"), "random", False,
     dict(vis_mut=dict(piv_le=True))),
    ("pivot bias omitted", (320, 64, 3, 40, 2, "ref"), "random", False, dict(bias_mode="none")),
    ("pivot bias log(s / n_piv)", (320, 64, 3, 129, 2, "ref"), "random", False, dict(bias_mode="div")),
    ("first, partly visible band tile skipped, w = 64", (512, 64, 3, 96, 2, "ref"), "random", False,
     dict(drop_tile=(3, "band", 0))),
    ("last partial pivot tile skipped, n_piv = 129", (320, 64, 3, 129, 2, "desc"), "pivot", False,
     dict(drop_tile=(2, "piv", 1))),
    ("pivots skipped by a block straddling times * w", (320, 64, 3, 129, 2, "ref"), "random", False,
     dict(sees_pivots_first_query=True)),
    ("dropout scale twice", (320, 64, 3, 129, 2, "ref"), "random", True, dict(drop_scale_power=2)),
    ("pivot slot p reads band key p's keep bit", (320, 64, 3, 129, 2, "ref"), "pivot", True,
     dict(keep_slot_from_band=True)),
]


@pytest.mark.parametrize("name,case,order,dropout,mut", FWD_MUTATIONS, ids=[m[0] for m in FWD_MUTATIONS])
def test_forward_mutation_breaks_the_bound(name, case, order, dropout, mut):
    s, w, times, n_piv, heads, kind = case
    for std in STDS:
        q, k, v, pivots, keep, _ = _inputs(s, w, times, n_piv, heads, std, order, kind)
        kp, p = (keep, P_DROP) if dropout else (None, 0.0)
        r, _ = _fwd_ratios(q, k, v, pivots, w, times, kp, p, **mut)
        print("%s, score std %g: emulation / bound %.1f" % (name, std, r))
        assert r > 1.0, (name, std, r)


# (name, case, order, dropout, backward mutation): one of dq / dk / dv must exceed its bound at every scale
BWD_MUTATIONS = [
    ("band start +1", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(band_shift=1))),
    ("band start -1", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(band_shift=-1))),
    ("diagonal +1", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(diag=1))),
    ("diagonal -1", (256, 16, 2, 40, 2, "ref"), "random", False, dict(vis_mut=dict(diag=-1))),
    ("pivot test <= with pivots planted at band starts", (256, 16, 2, None, 2, "planted"), "random", False,
     dict(vis_mut=dict(piv_le=True))),
    ("pivot bias omitted in the pivot pass", (320, 64, 3, 40, 2, "ref"), "random", False, dict(bias_mode="none")),
    ("band pass one query block short", (320, 64, 3, 129, 2, "ref"), "random", False, dict(band_last_shift=-1)),
    ("pivot pass one query block late", (320, 64, 3, 129, 2, "ref"), "random", False, dict(piv_first_shift=1)),
    ("pivot scatter skipped", (320, 64, 3, 129, 2, "ref"), "pivot", False, dict(scatter="skip")),
    ("pivot scatter applied twice", (320, 64, 3, 129, 2, "ref"), "pivot", False, dict(scatter="twice")),
    ("pivot scatter onto position + 1", (320, 64, 3, 129, 2, "ref"), "pivot", False, dict(scatter="next")),
    ("dropout scale twice", (320, 64, 3, 129, 2, "ref"), "random", True, dict(drop_scale_power=2)),
]


@pytest.mark.parametrize("name,case,order,dropout,mut", BWD_MUTATIONS, ids=[m[0] for m in BWD_MUTATIONS])
def test_backward_mutation_breaks_the_bound(name, case, order, dropout, mut):
    s, w, times, n_piv, heads, kind = case
    for std in STDS:
        q, k, v, pivots, keep, d_out = _inputs(s, w, times, n_piv, heads, std, order, kind)
        kp, p = (keep, P_DROP) if dropout else (None, 0.0)
        r = _bwd_ratios(q, k, v, d_out, pivots, w, times, kp, p, **mut)
        print("%s, score std %g: emulation / bound dq %.1f dk %.1f dv %.1f" % ((name, std) + r))
        assert max(r) > 1.0, (name, std, r)
