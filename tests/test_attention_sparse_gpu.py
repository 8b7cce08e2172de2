"""Sparse attention checked element by element against a float64 reference: training (cv_attn_sparse_fwd /
cv_attn_sparse_bwd, is_sparse = 1) and inference (cv_attn_gather, cv_attn_decode_gather, is_sparse = 2).

The training attention of one batch row is dense attention over s + n_piv virtual keys (the sequence, then the gathered
pivots; tests/attention_ref.py), so it gets dense attention's bf16 error model, u = 2^-8:
    out  |out - ref| <= 2u |ref| + u (P |V|) + 1e-5            lse  |lse - ref| <= 2u + 1e-5
    dX   |dX - ref| <= u |ref| + 2u (the same product on absolute values) + 1e-5, and at a pivot position the bound of
         its band part + the bound of its pivot slot + u (|band part| + |slot part|): the two parts are rounded to bf16
         separately and their sum once more.
tests/test_attention_sparse_bounds_cpu.py derives the bounds and shows that a kernel off by one key at a window edge,
one pivot, one tile of its walk, the pivot bias, the scatter or a dropout scale breaks them.  The cases sit on window
and tile edges: windows that do not divide 128, s = times * w (no query sees a pivot), n_piv at the pivot-tile edge,
pivots planted at band_start(i) - 1 and band_start(i) of window-edge queries.  Gathered decode attention gets the
forward bound over the gathered keys.  The float64 references run on the GPU one batch row at a time.
"""
import math
import random
import zlib

import pytest
import torch

import attention_ref as R
import sparse_dropout_ref as SD

pytestmark = pytest.mark.gpu

P_DROP = 0.1
BF = torch.bfloat16
# score standard deviation and key ordering (attention_ref.make_inputs); 'pivot' gives the pivot keys +6 std
VARIANTS = tuple((std, order) for order in ("random", "rising", "first", "pivot") for std in (1.0, 6.0))
BWD_VARIANTS = ((1.0, "random"), (6.0, "random"), (6.0, "pivot"))
WORST = {}


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module", autouse=True)
def _report_worst_ratios():
    yield
    if WORST:
        print("\nworst error / bound per test and output:")
        for key in sorted(WORST):
            print("  %-48s %-4s %.3f" % (key + (WORST[key],)))


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def _within(test, name, got, ref, bound, where):
    """Every element of got within bound of ref (NaN and inf fail); record the worst ratio."""
    r = (got.double() - ref).abs() / bound
    r = torch.where(torch.isfinite(r), r, torch.full_like(r, math.inf))
    worst = r.max().item() if r.numel() else 0.0
    if not worst <= 1.0:
        bad = (r > 1.0).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError("%s %s %s: %d elements outside the bound, first at %s: got %r, float64 %r, bound %.3g "
                             "(worst ratio %.3g)" % (test, name, where, bad.shape[0], i, got[i].item(), ref[i].item(),
                                                     bound[i].item(), worst))
    WORST[(test, name)] = max(WORST.get((test, name), 0.0), worst)


# ----------------------------------------------------------------------------------------------------
# pivot sets
# ----------------------------------------------------------------------------------------------------
def _ref_pivots(b, s, n_piv, txt, seed):
    """The reference's order (mpu/sparse_transformer.py:557-565): row i's txt[i] text positions first, then
    random.sample of the other positions; a different set per row."""
    rnd = random.Random(seed)
    rows = []
    for i in range(b):
        t = min(txt[i % len(txt)], n_piv)
        rows.append(list(range(t)) + rnd.sample(range(t, s), n_piv - t))
    return torch.tensor(rows, dtype=torch.long)


def _planted_pivots(b, s, w, times, seed):
    """For the window-edge queries i = g*w and g*w - 1 the positions band_start(i) - 1 and band_start(i), plus 0, 127,
    128 and s - 1; the same set in a different order per row."""
    pos = {0, 127, 128, s - 1}
    for g in range(1, s // w + 1):
        for i in (g * w, g * w - 1):
            if i < s:
                bs = max(0, i // w - times + 1) * w
                pos |= {bs - 1, bs} if bs > 0 else set()
    base = sorted(x for x in pos if 0 <= x < s)
    rnd = random.Random(seed)
    return torch.tensor([rnd.sample(base, len(base)) for _ in range(b)], dtype=torch.long)


def _pivot_sets(b, s, w, times, n_piv, txt):
    return (("ref", _ref_pivots(b, s, n_piv, txt, s + n_piv)), ("planted", _planted_pivots(b, s, w, times, s)))


# ----------------------------------------------------------------------------------------------------
# references
# ----------------------------------------------------------------------------------------------------
def _check_fwd(test, q, k, v, heads, pivots, w, times, out, lse, where, keep=None, p=0.0):
    """q / k / v [b, s, h] views, pivots [b, n_piv] (cuda), out [b, s, h], lse [b, heads, s]; keep [b, heads, s,
    s + n_piv] over the virtual keys or None."""
    s, n_piv = q.shape[1], pivots.shape[1]
    bias = R.pivot_bias(s, n_piv, device=q.device)
    for bi in range(q.shape[0]):
        qh, kh, vh = (R.heads_of(t[bi:bi + 1], heads) for t in (q, k, v))
        vk = R.virtual_keys(vh, pivots[bi])
        kp = None if keep is None else keep[bi:bi + 1]
        ref, lse_ref, probs = R.forward64(qh, R.virtual_keys(kh, pivots[bi]), vk,
                                          R.sparse_visible(s, w, times, pivots[bi]), kp, p, bias)
        at = "%s batch %d" % (where, bi)
        _within(test, "out", R.heads_of(out[bi:bi + 1], heads), ref, R.fwd_bound(ref, probs, vk, kp, p), at)
        _within(test, "lse", lse[bi:bi + 1], lse_ref, torch.full_like(lse_ref, R.lse_bound()), at)


def _check_bwd(test, q, k, v, d_out, heads, pivots, w, times, dqkv, where, keep=None, p=0.0):
    s, h, n_piv = q.shape[1], q.shape[2], pivots.shape[1]
    bias = R.pivot_bias(s, n_piv, device=q.device)
    for bi in range(q.shape[0]):
        qh, kh, vh, dh = (R.heads_of(t[bi:bi + 1], heads) for t in (q, k, v, d_out))
        kp = None if keep is None else keep[bi:bi + 1]
        grads, bounds = R.sparse_backward64(qh, kh, vh, dh, pivots[bi], R.sparse_visible(s, w, times, pivots[bi]),
                                            bias, kp, p)
        for j, name in enumerate(("dq", "dk", "dv")):
            got = R.heads_of(dqkv[bi:bi + 1, :, j * h:(j + 1) * h], heads)
            _within(test, name, got, grads[j], bounds[j], "%s batch %d" % (where, bi))


def _packed(q, k, v):
    h = q.shape[2]
    qkv = torch.cat((q, k, v), dim=-1)
    return qkv[..., :h], qkv[..., h:2 * h], qkv[..., 2 * h:]


def _padded(t, extra_rows=3):
    """t [b, s, h] copied into a NaN-filled buffer with row stride 3h + 64 and batch stride (s + extra_rows) rows,
    starting 64 columns in: the returned view reads only what the kernel may read."""
    b, s, h = t.shape
    buf = torch.full((b, s + extra_rows, 3 * h + 64), float("nan"), dtype=BF, device=t.device)
    buf[:, :s, 64:64 + h] = t
    return buf[:, :s, 64:64 + h]


def _sparse_bwd(q, k, v, out, d_out, lse, heads, pivots, w, times, dropout_p=0.0, drop_mask=None):
    """cv_attn_sparse_bwd into a NaN-filled dqkv, so that an element the kernel never writes fails its bound."""
    from cogview_b200 import _lib
    b, s, h = q.shape
    n_piv = pivots.shape[1]
    dqkv = torch.full((b, s, 3 * h), float("nan"), dtype=BF, device=q.device)
    ws = torch.empty(_lib.lib().cv_attn_sparse_bwd_workspace_bytes(b, heads, 64, s, n_piv), dtype=torch.uint8,
                     device=q.device)
    rc = _lib.lib().cv_attn_sparse_bwd(_lib.ptr(q), q.stride(1), q.stride(0), _lib.ptr(k), k.stride(1), k.stride(0),
                                       _lib.ptr(v), v.stride(1), v.stride(0), _lib.ptr(pivots), _lib.ptr(out),
                                       _lib.ptr(d_out), _lib.ptr(lse), _lib.ptr(dqkv), _lib.ptr(ws), b, heads, 64, s,
                                       n_piv, w, times, float(dropout_p), _lib.ptr(drop_mask), _lib.stream_ptr())
    _lib.check(rc, "cv_attn_sparse_bwd")
    return dqkv


# ----------------------------------------------------------------------------------------------------
# forward
# ----------------------------------------------------------------------------------------------------
PAIRS = ((16, 4), (64, 1), (64, 3), (96, 2), (128, 2), (128, 6), (256, 2))
N_PIV_CYCLE = (1, 127, 128, 129, 300, None)                    # None: n_piv = s
SHAPES = ((1, 1), (2, 3), (3, 1), (1, 3), (2, 1), (3, 3))


def _lengths(w, times):
    """times*w (no query sees a pivot), times*w + w, a length that is not a multiple of 128 (when w allows one) and
    one of at least 1024, all multiples of w."""
    out = [times * w, times * w + w]
    if w % 128:
        out.append(next(m * w for m in range(times + 2, 10 ** 4) if (m * w) % 128))
        out.append(next(m * w for m in range(1, 10 ** 4) if m * w >= 1024 and (m * w) % 128))
    else:
        out.append(next(m * w for m in range(1, 10 ** 4) if m * w >= 1024 and m * w > out[1]))
    return sorted(set(out))


FWD_CASES = []
for _w, _times in PAIRS:
    for _s in _lengths(_w, _times):
        _n = N_PIV_CYCLE[len(FWD_CASES) % len(N_PIV_CYCLE)]
        FWD_CASES.append(SHAPES[len(FWD_CASES) % len(SHAPES)] + (_s, _w, _times, min(_n or _s, _s), (17, 0, 5)))
# the CogView-sr shape, the 4B model's 40 heads, and the cases of the earlier global-tolerance test
FWD_CASES += [(1, 2, 4096, 128, 6, 768, (100,)), (2, 40, 1088, 64, 3, 300, (17, 0)),
              (2, 3, 512, 64, 3, 96, (48, 20)), (1, 2, 1024, 128, 6, 200, (64,)), (2, 1, 256, 128, 2, 40, (0, 7)),
              (1, 1, 768, 128, 6, 64, (30,))]


@pytest.mark.parametrize("b,heads,s,w,times,n_piv,txt", FWD_CASES)
def test_forward_within_bound_at_window_and_tile_edges(ops, b, heads, s, w, times, n_piv, txt):
    """Packed QKV views [b, s, 3h] (the training layout); both pivot sets, every score scale and key ordering."""
    for kind, pivots in _pivot_sets(b, s, w, times, n_piv, txt):
        pivots = pivots.cuda()
        for std, order in VARIANTS:
            q, k, v = _packed(*R.make_inputs(b, heads, s, s, std, order, _gen(b, heads, s, w, times, kind, std, order),
                                             "cuda", pivots=pivots))
            out, lse = ops.attn_sparse_fwd(q, k, v, heads, pivots, w, times, want_lse=True)
            _check_fwd("forward", q, k, v, heads, pivots, w, times, out, lse,
                       "%s pivots (%d), std %g %s" % (kind, pivots.shape[1], std, order))


@pytest.mark.parametrize("b,heads,s,w,times,n_piv", [(2, 3, 320, 64, 3, 129), (3, 1, 288, 96, 2, 288)])
def test_forward_strided_views_write_nothing_outside_out_and_lse(ops, b, heads, s, w, times, n_piv):
    from cogview_b200 import _lib
    h = heads * 64
    pivots = _ref_pivots(b, s, n_piv, (5,), s).cuda()
    q, k, v = (_padded(t) for t in R.make_inputs(b, heads, s, s, 6.0, "pivot", _gen(b, heads, s, w, "strided"),
                                                 "cuda", pivots=pivots))
    ldo, bso, out_at, lse_at = h + 64, (s + 5) * (h + 64), 24, 40
    out_buf = torch.full((out_at + b * bso + 40,), 0x5A5A, dtype=torch.int16, device="cuda")
    lse_buf = torch.full((lse_at + b * heads * s + 40,), -12345.5, dtype=torch.float32, device="cuda")
    out = out_buf.view(BF).as_strided((b, s, h), (bso, ldo, 1), out_at)
    lse = lse_buf[lse_at:lse_at + b * heads * s]
    ws = torch.empty(_lib.lib().cv_attn_sparse_workspace_bytes(b, heads, 64, n_piv), dtype=torch.uint8, device="cuda")
    rc = _lib.lib().cv_attn_sparse_fwd(_lib.ptr(q), q.stride(1), q.stride(0), _lib.ptr(k), k.stride(1), k.stride(0),
                                       _lib.ptr(v), v.stride(1), v.stride(0), _lib.ptr(pivots), out.data_ptr(), ldo,
                                       bso, _lib.ptr(lse), _lib.ptr(ws), b, heads, 64, s, n_piv, w, times, 0.0, 0, 0,
                                       None, _lib.stream_ptr())
    _lib.check(rc, "cv_attn_sparse_fwd")
    inside = torch.zeros(out_buf.shape, dtype=torch.bool, device="cuda")
    inside.as_strided((b, s, h), (bso, ldo, 1), out_at).fill_(True)
    assert (out_buf[~inside] == 0x5A5A).all(), "cv_attn_sparse_fwd wrote outside its out view"
    assert (lse_buf[:lse_at] == -12345.5).all() and (lse_buf[lse_at + b * heads * s:] == -12345.5).all(), \
        "cv_attn_sparse_fwd wrote outside its lse"
    _check_fwd("forward_strided", q, k, v, heads, pivots, w, times, out, lse.view(b, heads, s), "strided")


# ----------------------------------------------------------------------------------------------------
# backward: q / k / v in padded NaN-filled buffers, dqkv NaN-filled
# ----------------------------------------------------------------------------------------------------
BWD_CASES = [c for i, c in enumerate(FWD_CASES[:-6]) if i % 2 == 0 or c[2] == c[3] * c[4]]
BWD_CASES += FWD_CASES[-6:]


@pytest.mark.parametrize("b,heads,s,w,times,n_piv,txt", BWD_CASES)
def test_backward_within_bound_at_window_and_tile_edges(ops, b, heads, s, w, times, n_piv, txt):
    """dq, dk, dv element by element, both pivot sets; a row written past s lands in the next batch element's padding
    or rows, and the NaN-filled dqkv catches a row never written."""
    h = heads * 64
    for kind, pivots in _pivot_sets(b, s, w, times, n_piv, txt):
        pivots = pivots.cuda()
        for std, order in BWD_VARIANTS:
            g = _gen(b, heads, s, w, times, kind, std, order, "bwd")
            q, k, v = (_padded(t) for t in R.make_inputs(b, heads, s, s, std, order, g, "cuda", pivots=pivots))
            d_out = torch.randn((b, s, h), generator=g, device="cuda").to(BF)
            out, lse = ops.attn_sparse_fwd(q, k, v, heads, pivots, w, times, want_lse=True)
            dqkv = _sparse_bwd(q, k, v, out, d_out, lse, heads, pivots, w, times)
            _check_bwd("backward", q, k, v, d_out, heads, pivots, w, times, dqkv,
                       "%s pivots (%d), std %g %s" % (kind, pivots.shape[1], std, order))


# ----------------------------------------------------------------------------------------------------
# attention-probability dropout: the reference is fed the kernel's own keep bits
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,heads,s,w,times,n_piv,txt", [(2, 3, 512, 64, 3, 96, (48, 20)),
                                                         (1, 2, 1024, 128, 6, 200, (64,)),
                                                         (1, 2, 4096, 128, 6, 768, (100,)),
                                                         (2, 1, 256, 128, 2, 40, (0, 7)),
                                                         (2, 2, 576, 96, 2, 129, (10, 3))])
def test_dropout_forward_backward_within_bound(ops, b, heads, s, w, times, n_piv, txt):
    h = heads * 64
    g = _gen(b, heads, s, w, times, "dropout")
    pivots = _ref_pivots(b, s, n_piv, txt, 99).cuda()
    q, k, v = _packed(*R.make_inputs(b, heads, s, s, 1.0, "pivot", g, "cuda", pivots=pivots))
    d_out = torch.randn((b, s, h), generator=g, device="cuda").to(BF)
    args = (q, k, v, heads, pivots, w, times)
    out, lse, mask = ops.attn_sparse_fwd(*args, want_lse=True, dropout=(P_DROP, 1234, 7))
    dqkv = _sparse_bwd(q, k, v, out, d_out, lse, heads, pivots, w, times, P_DROP, mask)
    assert torch.equal(ops.attn_sparse_fwd(*args, dropout=None), ops.attn_sparse_fwd(*args)), \
        "dropout off is not the kernel without dropout, bit for bit"
    _, mask2 = ops.attn_sparse_fwd(*args, dropout=(P_DROP, 1234, 8))
    fwd, bwd = SD.decode_keep(mask, b, heads, s, n_piv, w, times)
    vis = SD.visible(s, n_piv, w, times, pivots.cpu()).unsqueeze(1).expand_as(fwd)
    assert (fwd[vis] >= 0).all() and (bwd[vis] >= 0).all(), "a visible pair has no keep bit"
    both = (fwd >= 0) & (bwd >= 0)
    assert torch.equal(fwd[both], bwd[both]), "forward and backward layouts disagree"
    fwd2, _ = SD.decode_keep(mask2, b, heads, s, n_piv, w, times)
    assert (fwd2[vis] != fwd[vis]).float().mean().item() > 0.1, "another site gives the same mask"
    nkb = (s + 127) // 128
    keep = torch.cat((fwd[..., :s], fwd[..., nkb * 128:nkb * 128 + n_piv]), -1).clamp_min(0).cuda()
    _check_fwd("dropout_forward", q, k, v, heads, pivots, w, times, out, lse, "dropout", keep, P_DROP)
    _check_bwd("dropout_backward", q, k, v, d_out, heads, pivots, w, times, dqkv, "dropout", keep, P_DROP)


# ----------------------------------------------------------------------------------------------------
# host-side refusals: arguments the kernels do not support fail before any launch, outputs untouched
# ----------------------------------------------------------------------------------------------------
def test_host_side_refusals(ops):
    from cogview_b200 import _lib
    lib = _lib.lib()
    s, h, w, times, n_piv = 128, 64, 64, 1, 4
    qkv = torch.zeros((1, s, 3 * h), dtype=BF, device="cuda")
    pivots = torch.zeros((1, n_piv), dtype=torch.long, device="cuda")
    out = torch.full((1, s, h), 7.0, dtype=BF, device="cuda")
    lse = torch.full((1, 1, s), 7.0, dtype=torch.float32, device="cuda")
    dqkv = torch.full((1, s, 3 * h), 7.0, dtype=BF, device="cuda")
    ws = torch.zeros(lib.cv_attn_sparse_bwd_workspace_bytes(1, 1, 64, s, s), dtype=torch.uint8, device="cuda")
    q, k, v = qkv.data_ptr(), qkv.data_ptr() + 2 * h, qkv.data_ptr() + 4 * h

    def fwd(n=n_piv, win=w, ld=3 * h, head_dim=64, p=0.0):
        return lib.cv_attn_sparse_fwd(q, ld, s * 3 * h, k, ld, s * 3 * h, v, ld, s * 3 * h, pivots.data_ptr(),
                                      out.data_ptr(), h, s * h, lse.data_ptr(), ws.data_ptr(), 1, 1, head_dim, s, n,
                                      win, times, p, 0, 0, None, _lib.stream_ptr())

    def bwd(n=n_piv, win=w, ld=3 * h, head_dim=64, p=0.0):
        return lib.cv_attn_sparse_bwd(q, ld, s * 3 * h, k, ld, s * 3 * h, v, ld, s * 3 * h, pivots.data_ptr(),
                                      out.data_ptr(), out.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), ws.data_ptr(),
                                      1, 1, head_dim, s, n, win, times, p, None, _lib.stream_ptr())

    refusals = []
    for name, call in (("forward", fwd), ("backward", bwd)):
        refusals += [(name + " s % w != 0", lambda c=call: c(win=96), "multiple of query_window"),
                     (name + " n_piv = 0", lambda c=call: c(n=0), "bad sizes"),
                     (name + " n_piv > s", lambda c=call: c(n=s + 1), "bad sizes"),
                     (name + " head_dim 32", lambda c=call: c(head_dim=32), "head_dim"),
                     (name + " dropout without a mask", lambda c=call: c(p=0.1), "keep.mask"),
                     (name + " row stride not a multiple of 8", lambda c=call: c(ld=3 * h + 4), "multiples of 8")]
    for name, call, message in refusals:
        with pytest.raises(_lib.CogViewB200Error, match=message):
            _lib.check(call(), name)
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (lse == 7.0).all() and (dqkv == 7.0).all(), "a refused call wrote its outputs"


# ----------------------------------------------------------------------------------------------------
# sparse inference: attention over a gathered key list of the K|V cache
# ----------------------------------------------------------------------------------------------------
def _gather_ref(q, cache, idx, heads, sq):
    """float64 softmax over K[idx], V[idx] of one row, -10000 above the diagonal of the last sq x sq block."""
    h = heads * 64
    n = idx.shape[0]
    kk, vv = (R.heads_of(cache[None, idx, o:o + h], heads) for o in (0, h))
    i = torch.arange(sq, device=q.device)[:, None]
    j = torch.arange(n, device=q.device)[None, :]
    vis = (j - (n - sq)) <= i
    ref, _, probs = R.forward64(R.heads_of(q[None], heads), kk, vv, vis)
    return ref, R.fwd_bound(ref, probs, vv)


GATHER_CASES = [(sq, n) for sq in (1, 2, 17, 64, 65) for n in sorted({sq, sq + 1, 63, 64, 65, 1001}) if n >= sq]


@pytest.mark.parametrize("sq,n", GATHER_CASES)
def test_attn_gather_within_bound(ops, sq, n):
    """cv_attn_gather: an index list in arbitrary order; every cache slot outside it is NaN."""
    b, heads = ((1, 1), (2, 3), (3, 2))[(sq + n) % 3]
    h, max_len = heads * 64, 1100
    g = _gen(sq, n, "gather")
    cache = torch.full((b, max_len, 2 * h), float("nan"), dtype=BF, device="cuda")
    idx = torch.stack([torch.randperm(max_len, generator=g, device="cuda")[:n] for _ in range(b)])
    for std, order in ((1.0, "random"), (6.0, "random")):
        q, k, v = R.make_inputs(b, heads, sq, n, std, order, _gen(sq, n, std), "cuda")
        for bi in range(b):
            cache[bi, idx[bi], :h], cache[bi, idx[bi], h:] = k[bi], v[bi]
        q = torch.cat((q, q, q), dim=-1)[..., :h]                      # a [b, sq, 3h] view, as the QKV GEMM leaves it
        out = ops.attn_gather(q, cache, idx, heads)
        for bi in range(b):
            ref, bound = _gather_ref(q[bi], cache[bi], idx[bi], heads, sq)
            _within("gather", "out", R.heads_of(out[bi:bi + 1], heads), ref, bound,
                    "std %g batch %d" % (std, bi))


# the cases of the earlier global-tolerance test ((b, heads, t, n, nsplit) = (2, 4, 300, 150, 1), (4, 40, 1000, 896, 8),
# (1, 8, 64, 65, 4)) are (t, nsplit) = (300, 1), (1000, 8), (64, 4) with their n cached keys
DECODE_CASES = [(t, nsplit) for t in (0, 1, 63, 64, 1087) for nsplit in (1, 2, 8, 64)]
DECODE_CASES += [(300, 1), (1000, 8), (64, 4)]
DECODE_KEYS = {0: 0, 1: 1, 63: 63, 64: 64, 1087: 700, 300: 149, 1000: 895}
DECODE_SHAPES = {1000: (4, 40), 300: (2, 4), 64: (1, 8)}


@pytest.mark.parametrize("t,nsplit", DECODE_CASES)
def test_attn_decode_gather_within_bound(ops, t, nsplit):
    """cv_attn_decode_gather with the new token's position t first, in the middle and last in the list; idx entries
    past *n_dev name a valid slot that is not listed and holds NaN.  The new K|V lands bitwise at slot t and no other
    cache byte changes."""
    b, heads = DECODE_SHAPES.get(t, ((1, 1), (2, 3), (3, 2))[(t + nsplit) % 3])
    h, max_len = heads * 64, 1100
    for where in ("first", "middle", "last"):
        g = _gen(t, nsplit, where, "decode")
        cache = torch.full((b, max_len, 2 * h), float("nan"), dtype=BF, device="cuda")
        prev = torch.stack([torch.randperm(t, generator=g, device="cuda")[:DECODE_KEYS[t]] for _ in range(b)])
        n = prev.shape[1] + 1
        at = {"first": 0, "middle": n // 2, "last": n - 1}[where]
        tt = torch.full((b, 1), t, dtype=torch.long, device="cuda")
        lst = torch.cat((prev[:, :at], tt, prev[:, at:]), dim=1)
        q, k, v = R.make_inputs(b, heads, 1, max_len, 1.0 if nsplit % 2 else 6.0, "random", g, "cuda")
        for bi in range(b):
            cache[bi, prev[bi], :h], cache[bi, prev[bi], h:] = k[bi, prev[bi]], v[bi, prev[bi]]
        qkv = torch.cat((q[:, 0], k[:, t], v[:, t]), dim=-1).contiguous()
        idx = torch.full((b, n + 5), max_len - 1, dtype=torch.int32, device="cuda")
        idx[:, :n] = lst.to(torch.int32)
        before = cache.clone()
        out = ops.attn_decode_gather(qkv, cache, heads, torch.tensor([t], dtype=torch.int32, device="cuda"), idx,
                                     torch.tensor([n], dtype=torch.int32, device="cuda"), nsplit=nsplit)
        bits, bits0 = cache.view(torch.int16), before.view(torch.int16)
        assert torch.equal(bits[:, t], qkv[:, h:].view(torch.int16)), "the new K|V is not at slot t"
        assert torch.equal(torch.cat((bits[:, :t], bits[:, t + 1:]), 1), torch.cat((bits0[:, :t], bits0[:, t + 1:]), 1)), \
            "a cache byte outside slot t changed"
        for bi in range(b):
            ref, bound = _gather_ref(q[bi], cache[bi], lst[bi], heads, 1)
            _within("decode_gather", "out", R.heads_of(out[bi:bi + 1, None], heads), ref, bound,
                    "t %d at %s, batch %d" % (t, where, bi))
