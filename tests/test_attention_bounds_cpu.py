"""The per-element error bounds of dense attention (tests/attention_ref.py) are the yardstick of
tests/test_attention_dense_gpu.py.  These CPU tests are the argument that the yardstick is right:

* an emulation of the kernels' own rounding (fp32 scores and accumulators, online softmax over 128-key tiles, bf16 P
  in the P V product and the row sum, bf16 dS and outputs) stays within 0.75 of every bound, at the score scales and
  key orderings the GPU test uses;
* the same emulation with one plausible kernel bug (`sep` or the causal diagonal or `off = sk - sq` moved by one key,
  a key tile skipped where it holds visible keys, the dropout scale applied twice) exceeds the bound on the same
  inputs, so a kernel with that bug would fail the GPU test.

The forward bound is a worst case to first order in u: every bf16 rounding of P and of the output is at most u.  With
dropout the emulation can reach 0.81 of it on other seeds (a row whose largest probability is dropped, leaving two
kept terms that cancel, each rounded the same way), so dropout forwards are held to 0.85 instead of 0.75; that is the
model being tight, not a missed rounding source.
"""
import pytest
import torch

import attention_ref as R

P_DROP = 0.1
STDS = (1.0, 6.0)
ORDERS = ("random", "rising", "first")
# (b, heads, sq, sk, sep): sep at a tile edge, causal with partial last tiles, memory (sq < sk) with sep > 0 and a
# long memory whose sep ends on a tile edge
CASES = [(1, 2, 300, 300, 129), (1, 2, 300, 300, 0), (1, 2, 257, 257, 0), (1, 2, 200, 328, 40), (1, 1, 129, 1100, 128)]


def _inputs(b, heads, sq, sk, sep, std, order, seed=0):
    g = torch.Generator().manual_seed(1000 * sq + sk + 7 * sep + int(std) + seed)
    q, k, v = (R.heads_of(t, heads) for t in R.make_inputs(b, heads, sq, sk, std, order, g))
    keep = torch.rand((b, heads, sq, sk), generator=g) >= P_DROP
    d_out = torch.randn((b, heads, sq, 64), generator=g).to(torch.bfloat16)
    return q, k, v, keep, d_out


def _fwd_ratios(q, k, v, sep, keep, p, *, diag=0, sep_shift=0, off_shift=0, drop_tile=None, drop_scale_power=1):
    """Worst (out, lse) ratios of the emulated forward (mutated as asked) against the float64 reference."""
    sq, sk = q.shape[-2], k.shape[-2]
    vis = R.visible(sq, sk, sep, diag=diag, sep_shift=sep_shift, off_shift=off_shift)
    out, lse = R.emulate_fwd(q, k, v, vis, keep, p, drop_tile=drop_tile, drop_scale_power=drop_scale_power)
    ref, lse_ref, probs = R.forward64(q, k, v, R.visible(sq, sk, sep), keep, p)
    return R.ratio(out, ref, R.fwd_bound(ref, probs, v, keep, p)), R.ratio(lse, lse_ref, R.lse_bound())


def _bwd_ratios(q, k, v, d_out, sep, keep, p, *, diag=0, sep_shift=0, drop_tile=None, drop_scale_power=1):
    """Worst (dq, dk, dv) ratios of the emulated backward (mutated as asked; the forward it is given is correct)."""
    s = q.shape[-2]
    vis_ref = R.visible(s, s, sep)
    out, lse = R.emulate_fwd(q, k, v, vis_ref, keep, p)
    vis = R.visible(s, s, sep, diag=diag, sep_shift=sep_shift)
    got = R.emulate_bwd(q, k, v, out, d_out, lse, vis, keep, p, drop_tile=drop_tile,
                        drop_scale_power=drop_scale_power)
    grads, ref_out, probs = R.backward64(q, k, v, d_out, vis_ref, keep, p)
    bounds = R.bwd_bounds(q, k, v, d_out, ref_out, probs, grads, keep, p)
    return tuple(R.ratio(gt, gr, bd) for gt, gr, bd in zip(got, grads, bounds))


@pytest.mark.parametrize("b,heads,sq,sk,sep", CASES)
def test_emulated_kernels_stay_within_the_bounds(b, heads, sq, sk, sep):
    worst = {}
    for std in STDS:
        for order in ORDERS:
            for dropout in (False, True):
                q, k, v, keep, d_out = _inputs(b, heads, sq, sk, sep, std, order)
                kp, p = (keep, P_DROP) if dropout else (None, 0.0)
                tag = "drop" if dropout else "nodrop"
                fo, fl = _fwd_ratios(q, k, v, sep, kp, p)
                worst["out_" + tag] = max(worst.get("out_" + tag, 0.0), fo)
                worst["lse"] = max(worst.get("lse", 0.0), fl)
                if sq == sk:
                    for name, r in zip(("dq", "dk", "dv"), _bwd_ratios(q, k, v, d_out, sep, kp, p)):
                        worst[name] = max(worst.get(name, 0.0), r)
    print("emulation / bound, worst over score std %s and orders %s:" % (STDS, ORDERS),
          " ".join("%s %.3f" % kv for kv in sorted(worst.items())))
    limits = {"out_drop": 0.85}
    for name, r in worst.items():
        assert r <= limits.get(name, 0.75), (name, r)


# (name, case, forward mutation): each must push the emulated forward past the bound at every score scale
FWD_MUTATIONS = [
    ("sep+1", (1, 2, 300, 300, 129), dict(sep_shift=1)),
    ("sep-1", (1, 2, 300, 300, 129), dict(sep_shift=-1)),
    ("sep+1 with memory", (1, 2, 200, 328, 40), dict(sep_shift=1)),
    ("sep-1 with memory", (1, 2, 200, 328, 40), dict(sep_shift=-1)),
    ("diagonal+1", (1, 2, 257, 257, 0), dict(diag=1)),
    ("diagonal-1", (1, 2, 257, 257, 0), dict(diag=-1)),
    ("diagonal+1 with memory", (1, 2, 200, 328, 40), dict(diag=1)),
    ("diagonal-1 with memory", (1, 2, 200, 328, 40), dict(diag=-1)),
    ("off+1", (1, 2, 200, 328, 40), dict(off_shift=1)),
    ("off-1", (1, 2, 200, 328, 40), dict(off_shift=-1)),
    ("off+1, long memory", (1, 1, 129, 1100, 128), dict(off_shift=1)),
    ("off-1, long memory", (1, 1, 129, 1100, 128), dict(off_shift=-1)),
    ("diagonal key tile of the last query block skipped", (1, 2, 300, 300, 0), dict(drop_tile=(2, 2))),
    ("key tile holding only sep keys skipped", (1, 2, 300, 300, 129), dict(drop_tile=(0, 1))),
    ("first key tile skipped with memory", (1, 2, 200, 328, 40), dict(drop_tile=(1, 0))),
]


@pytest.mark.parametrize("name,case,mut", FWD_MUTATIONS, ids=[m[0] for m in FWD_MUTATIONS])
def test_forward_mutation_breaks_the_bound(name, case, mut):
    b, heads, sq, sk, sep = case
    for std in STDS:
        q, k, v, _, _ = _inputs(b, heads, sq, sk, sep, std, "random")
        r, _ = _fwd_ratios(q, k, v, sep, None, 0.0, **mut)
        print("%s, score std %g: emulation / bound %.1f" % (name, std, r))
        assert r > 1.0, (name, std, r)


def test_forward_dropout_scale_twice_breaks_the_bound():
    b, heads, sq, sk, sep = 1, 2, 300, 300, 129
    for std in STDS:
        q, k, v, keep, _ = _inputs(b, heads, sq, sk, sep, std, "random")
        r, _ = _fwd_ratios(q, k, v, sep, keep, P_DROP, drop_scale_power=2)
        print("dropout scale twice, score std %g: emulation / bound %.1f" % (std, r))
        assert r > 1.0, (std, r)


# (name, (b, heads, s, sep), backward mutation, dropout): one of dq / dk / dv must exceed its bound at every scale
BWD_MUTATIONS = [
    ("sep+1", (1, 2, 300, 129), dict(sep_shift=1), False),
    ("sep-1", (1, 2, 300, 129), dict(sep_shift=-1), False),
    ("diagonal+1", (1, 2, 257, 0), dict(diag=1), False),
    ("diagonal-1", (1, 2, 257, 0), dict(diag=-1), False),
    ("query block 0 skipped for a key block holding sep keys", (1, 2, 300, 256), dict(drop_tile=(0, 1)), False),
    ("diagonal tile of the last blocks skipped", (1, 2, 300, 0), dict(drop_tile=(2, 2)), False),
    ("dropout scale twice", (1, 2, 300, 129), dict(drop_scale_power=2), True),
]


@pytest.mark.parametrize("name,case,mut,dropout", BWD_MUTATIONS, ids=[m[0] for m in BWD_MUTATIONS])
def test_backward_mutation_breaks_the_bound(name, case, mut, dropout):
    b, heads, s, sep = case
    for std in STDS:
        q, k, v, keep, d_out = _inputs(b, heads, s, s, sep, std, "random")
        kp, p = (keep, P_DROP) if dropout else (None, 0.0)
        r = _bwd_ratios(q, k, v, d_out, sep, kp, p, **mut)
        print("%s, score std %g: emulation / bound dq %.1f dk %.1f dv %.1f" % ((name, std) + r))
        assert max(r) > 1.0, (name, std, r)
