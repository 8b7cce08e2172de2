"""Nucleus (top-p) sampling for more than one row, on the host: top_k_logits on [b, V] logits against its one-row
branch (the reference's), the row-wise helper top_p_logits (no boolean indexing, so a CUDA graph can capture it), and
which route filling_sequence takes with top_p > 0 (a stand-in model records the calls)."""
import pytest
import torch
from torch.overrides import TorchFunctionMode


def _logits(b, V, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((b, V), generator=g) * 2.0


@pytest.mark.parametrize("b", [2, 7])
@pytest.mark.parametrize("top_k", [0, 20])
@pytest.mark.parametrize("top_p", [0.1, 0.5, 0.9])
def test_rows_match_the_one_row_call(b, top_k, top_p):
    from cogview_b200.generation import sampling
    logits = _logits(b, 500, seed=b * 100 + top_k)
    out = sampling.top_k_logits(logits.clone(), top_k=top_k, top_p=top_p)
    assert out.shape == (b, 500)
    for r in range(b):
        one = sampling.top_k_logits(logits[r:r + 1].clone(), top_k=top_k, top_p=top_p)
        assert torch.equal(out[r:r + 1], one), r
    # and it filtered something: at most top_k survivors, at least one per row
    kept = torch.isfinite(out).sum(1)
    assert bool((kept >= 1).all()) and bool((kept < 500).all())
    if top_k:
        assert bool((kept <= top_k).all())


class _NoBoolIndex(TorchFunctionMode):
    """Fails on indexing or index_put with a boolean tensor (a host sync, not capturable in a CUDA graph)."""

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func in (torch.Tensor.__getitem__, torch.Tensor.__setitem__, torch.Tensor.index_put_,
                    torch.Tensor.index_put, torch.index_put, torch.Tensor.masked_select, torch.masked_select,
                    torch.Tensor.nonzero, torch.nonzero):
            idx = args[1] if len(args) > 1 else None
            items = idx if isinstance(idx, (tuple, list)) else (idx,)
            for it in items:
                assert not (torch.is_tensor(it) and it.dtype == torch.bool), "boolean indexing in %s" % func
            assert func not in (torch.Tensor.masked_select, torch.masked_select, torch.Tensor.nonzero, torch.nonzero)
        return func(*args, **kwargs)


def test_helper_uses_no_boolean_indexing_and_one_row_is_unchanged():
    from cogview_b200.generation import sampling
    logits = _logits(5, 300, seed=3)
    with _NoBoolIndex():
        out = sampling.top_p_logits(logits.clone(), 0.8)
    # the mode does catch boolean indexing
    with pytest.raises(AssertionError):
        with _NoBoolIndex():
            x = logits.clone()
            x[x > 0] = 0.0
    # each row: kept iff the mass strictly before it in descending order is <= top_p (float64 restatement)
    for r in range(5):
        p = torch.softmax(logits[r].double(), -1)
        ps, order = torch.sort(p, descending=True)
        before = torch.cumsum(ps, 0) - ps
        want = torch.zeros(300, dtype=torch.bool)
        want[order[before <= 0.8]] = True
        assert torch.equal(torch.isfinite(out[r]), want)
        assert torch.equal(out[r][want], logits[r][want])
    # a [1, V] call keeps the reference's one-row branch and gives the helper's answer for that row
    one = sampling.top_k_logits(logits[1:2].clone(), top_k=0, top_p=0.8)
    assert one.shape == (1, 300) and torch.equal(one, out[1:2])


# ----------------------------------------------------------------------------------------------------
# routing of filling_sequence
# ----------------------------------------------------------------------------------------------------
N_IMG = 8192


class StandIn:
    """A dense model on the K|V cache: random logits per call (seeded by the cache length); generate_run records its
    arguments and returns image codes."""

    def __init__(self, V):
        self.V = V
        self.calls = []
        self.runs = []

    def __call__(self, tokens, position_ids, attention_mask, txt, img, is_sparse, *mems):
        assert is_sparse == 0
        t_prev = mems[0].shape[1] if mems else 0
        b, sq = tokens.shape
        self.calls.append((b, sq))
        g = torch.Generator().manual_seed(t_prev)
        logits = torch.randn((b, sq, self.V), generator=g)
        mem = torch.zeros((b, t_prev + sq, 1))
        return (logits, mem)

    def generate_run(self, last_tokens, first_pos, mems, n_steps, temperature, top_k, invalid_slices, sparse=None,
                     row_pad=None, top_p=0.0):
        self.runs.append(dict(b=last_tokens.shape[0], n_steps=n_steps, top_k=top_k, top_p=top_p))
        b = last_tokens.shape[0]
        new = (torch.arange(n_steps).unsqueeze(0) + torch.arange(b).unsqueeze(1)) % N_IMG
        mem = torch.zeros((b, mems[0].shape[1] + n_steps, 1))
        return new, torch.zeros(b), [mem]


def _args(top_p, top_k=0):
    return type("A", (), dict(temperature=1.0, top_k=top_k, top_p=top_p, is_sparse=0,
                              img_tokenizer_num_tokens=N_IMG))


def _template(tok, nb, n_gen):
    text = list(range(N_IMG, N_IMG + 6))
    return torch.tensor([tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + [-nb] * n_gen)


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=N_IMG, txt_tokens=101)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


@pytest.mark.parametrize("nb,top_k", [(2, 0), (8, 200), (65, 0)])
def test_several_beams_with_top_p_use_generate_run(tok, nb, top_k):
    from cogview_b200.generation import sampling
    m = StandIn(tok.num_tokens)
    seq = _template(tok, nb, 10)
    with torch.no_grad():
        out = sampling.filling_sequence(m, seq, _args(0.9, top_k))
    assert out.shape == (nb, len(seq))
    # the first slot expands 1 -> nb beams on the host; the other nine run on the graph with the nucleus
    assert m.runs == [dict(b=nb, n_steps=9, top_k=top_k, top_p=0.9)]
    assert bool((out[:, len(seq) - 10:] < N_IMG).all())


def test_several_beams_fall_back_to_the_batched_host_loop(tok):
    """When generate_run declines (graph off, more than 64 rows), the beams run on the host loop: top_k_logits on
    [nb, V] logits, which raised before the row-wise helper."""
    from cogview_b200.generation import sampling

    class Declines(StandIn):
        def generate_run(self, *a, **kw):
            super().generate_run(*a, **kw)
            return None
    m = Declines(tok.num_tokens)
    seq = _template(tok, 4, 10)
    with torch.no_grad():
        out = sampling.filling_sequence(m, seq, _args(0.9, 20))
    assert out.shape == (4, len(seq))
    assert [r['n_steps'] for r in m.runs] == list(range(9, 1, -1)) and all(r['top_p'] == 0.9 for r in m.runs)
    assert m.calls[0] == (1, len(seq) - 10) and all(c == (4, 1) for c in m.calls[1:]) and len(m.calls) == 10
    assert bool((out[:, len(seq) - 10:] < N_IMG).all())


def test_one_row_with_top_p_keeps_the_host_loop(tok):
    from cogview_b200.generation import sampling
    seq = _template(tok, 1, 10)
    outs = []
    for _ in range(2):
        m = StandIn(tok.num_tokens)
        torch.manual_seed(5)
        with torch.no_grad():
            outs.append(sampling.filling_sequence(m, seq, _args(0.9)))
        assert not m.runs and len(m.calls) == 10
    assert outs[0].shape == (1, len(seq)) and torch.equal(outs[0], outs[1])
    # without top_p the same template runs on the graph
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        sampling.filling_sequence(m, seq, _args(0.0))
    assert m.runs == [dict(b=1, n_steps=9, top_k=0, top_p=0.0)]
