"""Dense attention (cv_attn_fwd / cv_attn_bwd) checked element by element against a float64 reference.

Every output element must lie within the bf16 error model of tests/attention_ref.py (its derivation, and the proof
that a kernel off by one key, one tile or one dropout scale breaks it, is tests/test_attention_bounds_cpu.py):
    out  |out - ref| <= 2u |ref| + u (P |V|) + 1e-5            lse  |lse - ref| <= 2u + 1e-5
    dX   |dX - ref| <= u |ref| + 2u (the same product on absolute values) + 1e-5,   u = 2^-8
A global max|err| / max|ref| hides one wrong row or one wrong key tile of a long sequence; a per-element bound does
not.  The cases sit on the kernels' 128-query / 128-key tile edges, on both sides of their unmasked fast path (whole
tiles below `sep` or the diagonal) and on the strides and buffers a caller may pass.  The float64 references are
computed on the GPU one batch row at a time.
"""
import math
import zlib

import pytest
import torch

import attention_ref as R

pytestmark = pytest.mark.gpu

P_DROP = 0.1
BF = torch.bfloat16
# score standard deviation and key ordering (attention_ref.make_inputs): i.i.d. scores, a running maximum that rises
# in every key tile (the online-softmax rescale every tile), and one that sits in the first tile
VARIANTS = ((1.0, "random"), (6.0, "random"), (1.0, "rising"), (6.0, "rising"), (1.0, "first"), (6.0, "first"))
BWD_VARIANTS = ((1.0, "random"), (6.0, "random"), (6.0, "rising"))
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


def _check_fwd(test, q, k, v, heads, sep, out, lse, where, keep=None, p=0.0):
    """q [b, sq, h], k / v [b, sk, h] (views), out [b, sq, h], lse [b, heads, sq] or None; keep [b, heads, sq, sk]."""
    sq, sk = q.shape[1], k.shape[1]
    vis = R.visible(sq, sk, sep, device=q.device)
    for bi in range(q.shape[0]):
        qh, kh, vh = (R.heads_of(t[bi:bi + 1], heads) for t in (q, k, v))
        kp = None if keep is None else keep[bi:bi + 1]
        ref, lse_ref, probs = R.forward64(qh, kh, vh, vis, kp, p)
        at = "%s batch %d" % (where, bi)
        _within(test, "out", R.heads_of(out[bi:bi + 1], heads), ref, R.fwd_bound(ref, probs, vh, kp, p), at)
        if lse is not None:
            _within(test, "lse", lse[bi:bi + 1], lse_ref, torch.full_like(lse_ref, R.lse_bound()), at)


def _check_bwd(test, q, k, v, d_out, heads, sep, dqkv, where, keep=None, p=0.0):
    s, h = q.shape[1], q.shape[2]
    vis = R.visible(s, s, sep, device=q.device)
    for bi in range(q.shape[0]):
        qh, kh, vh, dh = (R.heads_of(t[bi:bi + 1], heads) for t in (q, k, v, d_out))
        kp = None if keep is None else keep[bi:bi + 1]
        grads, ref_out, probs = R.backward64(qh, kh, vh, dh, vis, kp, p)
        bounds = R.bwd_bounds(qh, kh, vh, dh, ref_out, probs, grads, kp, p)
        for j, name in enumerate(("dq", "dk", "dv")):
            got = R.heads_of(dqkv[bi:bi + 1, :, j * h:(j + 1) * h], heads)
            _within(test, name, got, grads[j], bounds[j], "%s batch %d" % (where, bi))


def _padded(t, extra_rows=3):
    """t [b, s, h] copied into a NaN-filled buffer with row stride 3h + 64 and batch stride (s + extra_rows) rows,
    starting 64 columns in: the returned view reads only what the kernel may read."""
    b, s, h = t.shape
    buf = torch.full((b, s + extra_rows, 3 * h + 64), float("nan"), dtype=BF, device=t.device)
    buf[:, :s, 64:64 + h] = t
    return buf[:, :s, 64:64 + h]


def _attn_bwd(ops, q, k, v, out, d_out, lse, heads, sep, dropout_p=0.0, drop_mask=None):
    """cv_attn_bwd into a NaN-filled dqkv, so that an element the kernel never writes fails its bound."""
    from cogview_b200 import _lib
    b, s, h = q.shape
    dqkv = torch.full((b, s, 3 * h), float("nan"), dtype=BF, device=q.device)
    ws = torch.empty(_lib.lib().cv_attn_bwd_workspace_bytes(b, heads, 64, s) // 4, dtype=torch.float32,
                     device=q.device)
    rc = _lib.lib().cv_attn_bwd(_lib.ptr(q), q.stride(1), q.stride(0), _lib.ptr(k), k.stride(1), k.stride(0),
                                _lib.ptr(v), v.stride(1), v.stride(0), _lib.ptr(out), _lib.ptr(d_out), _lib.ptr(lse),
                                _lib.ptr(dqkv), _lib.ptr(ws), b, heads, 64, s, sep, float(dropout_p),
                                _lib.ptr(drop_mask), _lib.stream_ptr())
    _lib.check(rc, "cv_attn_bwd")
    return dqkv


def _seps(s, candidates):
    return sorted({x for x in candidates if 0 <= x <= s})


def _cycle(lengths, sep_candidates, shapes):
    cases = []
    for s in lengths:
        for sep in _seps(s, sep_candidates + (s - 1, s)):
            b, heads = shapes[len(cases) % len(shapes)]
            cases.append((b, heads, s, sep))
    return cases


# ----------------------------------------------------------------------------------------------------
# forward, sq == sk
# ----------------------------------------------------------------------------------------------------
FWD_CASES = _cycle((1, 2, 63, 64, 65, 127, 128, 129, 255, 257, 1088, 1089), (0, 1, 2, 127, 128, 129),
                   ((1, 1), (3, 1), (1, 3), (3, 3)))
# the 4B model's training shape, and the cases of the earlier global-tolerance test
FWD_CASES += [(2, 40, 1088, 64), (2, 4, 128, 0), (2, 3, 200, 0), (1, 2, 1088, 0), (2, 2, 128, 40), (1, 2, 300, 130)]


@pytest.mark.parametrize("b,heads,s,sep", FWD_CASES)
def test_forward_within_bound_at_tile_and_mask_edges(ops, b, heads, s, sep):
    """Packed QKV views [b, s, 3h] (the training layout); every score scale and key ordering of VARIANTS."""
    h = heads * 64
    for std, order in VARIANTS:
        q, k, v = R.make_inputs(b, heads, s, s, std, order, _gen(b, heads, s, sep, std, order), "cuda")
        qkv = torch.cat((q, k, v), dim=-1)
        q, k, v = qkv[..., :h], qkv[..., h:2 * h], qkv[..., 2 * h:]
        out, lse = ops.attn_fwd(q, k, v, heads, sep=sep, want_lse=True)
        _check_fwd("forward", q, k, v, heads, sep, out, lse, "std %g %s" % (std, order))


# ----------------------------------------------------------------------------------------------------
# forward with memory, sq < sk: K / V are views of a longer K|V cache whose unused slots are NaN
# ----------------------------------------------------------------------------------------------------
MEM_CASES = []
for _off in (1, 127, 128, 129, 971):
    for _sq in (1, 64, 129, 200):
        for _sep in _seps(_sq, (0, 1, 128, _sq)):
            MEM_CASES.append(((1, 1), (2, 3), (3, 1), (1, 2))[len(MEM_CASES) % 4] + (_sq, _sq + _off, _sep))
MEM_CASES.append((2, 2, 72, 200, 0))        # the earlier global-tolerance test's memory case


@pytest.mark.parametrize("b,heads,sq,sk,sep", MEM_CASES)
def test_forward_with_memory_reads_only_the_first_sk_cache_slots(ops, b, heads, sq, sk, sep):
    h = heads * 64
    max_len = sk + 72
    for std, order in ((1.0, "random"), (6.0, "random"), (6.0, "rising")):
        q, k, v = R.make_inputs(b, heads, sq, sk, std, order, _gen(b, heads, sq, sk, sep, std, order), "cuda")
        cache = torch.full((b, max_len, 2 * h), float("nan"), dtype=BF, device="cuda")
        cache[:, :sk, :h], cache[:, :sk, h:] = k, v
        k, v = cache[:, :sk, :h], cache[:, :sk, h:]
        out, lse = ops.attn_fwd(q, k, v, heads, sep=sep, want_lse=True)
        assert torch.isfinite(out).all() and torch.isfinite(lse).all()
        _check_fwd("forward_memory", q, k, v, heads, sep, out, lse, "std %g %s" % (std, order))


# ----------------------------------------------------------------------------------------------------
# strides: separate padded inputs, an out view with padded row and batch strides, lse at an offset
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,heads,sq,sk,sep", [(2, 3, 129, 129, 128), (2, 2, 65, 200, 1), (3, 1, 257, 257, 0)])
def test_forward_strided_views_write_nothing_outside_out_and_lse(ops, b, heads, sq, sk, sep):
    from cogview_b200 import _lib
    h = heads * 64
    q, k, v = (_padded(t) for t in R.make_inputs(b, heads, sq, sk, 6.0, "random", _gen(b, heads, sq, sk, sep),
                                                 "cuda"))
    ldo, bso, out_at, lse_at = h + 64, (sq + 5) * (h + 64), 24, 40
    out_buf = torch.full((out_at + b * bso + 40,), 0x5A5A, dtype=torch.int16, device="cuda")
    lse_buf = torch.full((lse_at + b * heads * sq + 40,), -12345.5, dtype=torch.float32, device="cuda")
    out = out_buf.view(BF).as_strided((b, sq, h), (bso, ldo, 1), out_at)
    lse = lse_buf[lse_at:lse_at + b * heads * sq]
    rc = _lib.lib().cv_attn_fwd(_lib.ptr(q), q.stride(1), q.stride(0), _lib.ptr(k), k.stride(1), k.stride(0),
                                _lib.ptr(v), v.stride(1), v.stride(0), out.data_ptr(), ldo, bso, _lib.ptr(lse), b,
                                heads, 64, sq, sk, sep, 0.0, 0, 0, None, _lib.stream_ptr())
    _lib.check(rc, "cv_attn_fwd")
    inside = torch.zeros(out_buf.shape, dtype=torch.bool, device="cuda")
    inside.as_strided((b, sq, h), (bso, ldo, 1), out_at).fill_(True)
    assert (out_buf[~inside] == 0x5A5A).all(), "cv_attn_fwd wrote outside its out view"
    assert (lse_buf[:lse_at] == -12345.5).all() and (lse_buf[lse_at + b * heads * sq:] == -12345.5).all(), \
        "cv_attn_fwd wrote outside its lse"
    _check_fwd("forward_strided", q, k, v, heads, sep, out, lse.view(b, heads, sq), "strided")


# ----------------------------------------------------------------------------------------------------
# backward (sq == sk)
# ----------------------------------------------------------------------------------------------------
BWD_CASES = [c + ("packed",) for c in _cycle((1, 64, 127, 128, 129, 257, 300, 1088), (0, 1, 127, 128, 129, 256),
                                             ((1, 1), (2, 1), (1, 3), (2, 3)))]
# the 4B model's training shape, the cases of the earlier global-tolerance test, and padded separate inputs
BWD_CASES += [(2, 40, 1088, 0, "packed"), (2, 40, 1088, 64, "packed"), (2, 2, 128, 0, "packed"),
              (1, 3, 200, 0, "packed"), (2, 2, 384, 0, "packed"), (1, 2, 300, 130, "packed"),
              (1, 2, 1088, 0, "packed"), (2, 3, 300, 129, "padded"), (2, 1, 257, 0, "padded")]


@pytest.mark.parametrize("b,heads,s,sep,layout", BWD_CASES)
def test_backward_within_bound_at_tile_and_mask_edges(ops, b, heads, s, sep, layout):
    """dq, dk, dv element by element (with b = 2 and s % 128 != 0 a row written past s lands in the next batch
    element, and the NaN-filled dqkv catches a row never written)."""
    h = heads * 64
    for std, order in BWD_VARIANTS:
        g = _gen(b, heads, s, sep, layout, std, order)
        q, k, v = R.make_inputs(b, heads, s, s, std, order, g, "cuda")
        d_out = torch.randn((b, s, h), generator=g, device="cuda").to(BF)
        if layout == "packed":
            qkv = torch.cat((q, k, v), dim=-1)
            q, k, v = qkv[..., :h], qkv[..., h:2 * h], qkv[..., 2 * h:]
        else:
            q, k, v = _padded(q), _padded(k), _padded(v)
        out, lse = ops.attn_fwd(q, k, v, heads, sep=sep, want_lse=True)
        dqkv = _attn_bwd(ops, q, k, v, out, d_out, lse, heads, sep)
        _check_bwd("backward", q, k, v, d_out, heads, sep, dqkv, "std %g %s" % (std, order))


# ----------------------------------------------------------------------------------------------------
# attention-probability dropout: the reference is fed the kernel's own keep bits
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,heads,sq,sk,sep", [(2, 2, 129, 129, 0), (2, 2, 129, 129, 129), (2, 2, 300, 300, 0),
                                               (2, 2, 300, 300, 129), (2, 2, 129, 300, 128)])
def test_dropout_forward_backward_within_bound(ops, b, heads, sq, sk, sep):
    h = heads * 64
    g = _gen(b, heads, sq, sk, sep, "dropout")
    q, k, v = R.make_inputs(b, heads, sq, sk, 1.0, "random", g, "cuda")
    qkv = torch.cat((q, k, v), dim=-1) if sq == sk else None
    if qkv is not None:
        q, k, v = qkv[..., :h], qkv[..., h:2 * h], qkv[..., 2 * h:]
    out, lse, mask = ops.attn_fwd(q, k, v, heads, sep=sep, want_lse=True, dropout=(P_DROP, 4242, 17))
    keep_k, keep_q = R.keep_from_bits(mask, sq, sk)
    visited = R.visited_tiles(sq, sk, sep, device="cuda")
    assert torch.equal(keep_k * visited, keep_q * visited), "the two keep-bit layouts disagree"
    keep = keep_q * visited                  # bits outside the visited tiles are never written (and never visible)
    vis = R.visible(sq, sk, sep, device="cuda")
    rate = (keep * vis).sum().item() / (vis.sum().item() * b * heads)
    assert abs(rate - (1 - P_DROP)) < 0.02, rate
    _check_fwd("dropout_forward", q, k, v, heads, sep, out, lse, "dropout", keep, P_DROP)
    if sq == sk:
        d_out = torch.randn((b, sq, h), generator=g, device="cuda").to(BF)
        dqkv = _attn_bwd(ops, q, k, v, out, d_out, lse, heads, sep, P_DROP, mask)
        _check_bwd("dropout_backward", q, k, v, d_out, heads, sep, dqkv, "dropout", keep, P_DROP)


# ----------------------------------------------------------------------------------------------------
# host-side refusals: arguments the kernels do not support fail before any launch
# ----------------------------------------------------------------------------------------------------
def test_host_side_refusals(ops):
    from cogview_b200 import _lib
    lib = _lib.lib()
    s, h = 64, 64
    qkv = torch.zeros((1, s, 3 * h), dtype=BF, device="cuda")
    out = torch.zeros((1, s, h), dtype=BF, device="cuda")
    lse = torch.zeros((1, 1, s), dtype=torch.float32, device="cuda")
    dqkv = torch.zeros((1, s, 3 * h), dtype=BF, device="cuda")
    ws = torch.zeros(lib.cv_attn_bwd_workspace_bytes(1, 1, 64, s) // 4, dtype=torch.float32, device="cuda")
    q, k, v = qkv.data_ptr(), qkv.data_ptr() + 2 * h, qkv.data_ptr() + 4 * h

    def fwd(sq=s, sk=s, sep=0, ld=3 * h, head_dim=64, p=0.0):
        return lib.cv_attn_fwd(q, ld, s * 3 * h, k, ld, s * 3 * h, v, ld, s * 3 * h, out.data_ptr(), h, s * h,
                               lse.data_ptr(), 1, 1, head_dim, sq, sk, sep, p, 0, 0, None, _lib.stream_ptr())

    def bwd(sep=0, ld=3 * h, head_dim=64, p=0.0):
        return lib.cv_attn_bwd(q, ld, s * 3 * h, k, ld, s * 3 * h, v, ld, s * 3 * h, out.data_ptr(), out.data_ptr(),
                               lse.data_ptr(), dqkv.data_ptr(), ws.data_ptr(), 1, 1, head_dim, s, sep, p, None,
                               _lib.stream_ptr())

    refusals = [("sep > sq", lambda: fwd(sep=s + 1), "sep"),
                ("sk < sq", lambda: fwd(sq=s, sk=s - 1), "sk >= sq"),
                ("row stride not a multiple of 8", lambda: fwd(ld=3 * h + 4), "multiples of 8"),
                ("head_dim 32", lambda: fwd(head_dim=32), "head_dim"),
                ("dropout without a mask buffer", lambda: fwd(p=0.1), "keep-mask"),
                ("backward sep > s", lambda: bwd(sep=s + 1), "bad sizes"),
                ("backward row stride not a multiple of 8", lambda: bwd(ld=3 * h + 4), "multiples of 8"),
                ("backward head_dim 32", lambda: bwd(head_dim=32), "head_dim"),
                ("backward dropout without the keep mask", lambda: bwd(p=0.1), "keep mask")]
    for name, call, message in refusals:
        with pytest.raises(_lib.CogViewB200Error, match=message):
            _lib.check(call(), name)
    torch.cuda.synchronize()
