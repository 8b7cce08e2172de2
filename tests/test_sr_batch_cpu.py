"""Host side of super-resolving many images in one decode batch, with stand-in models: which template lists
filling_sequences runs as interleaved (given / generated stretches) batches and which it fills one by one, the per-row
positions of the chunks and generate runs ([ROI2] offsets differ per row), where the drawn tokens land, and
magnify_batch against magnify with a stand-in fill."""
import types

import pytest
import torch

N_IMG, N_TXT = 8192, 101
H, L = 4, 2


class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 200, 0.0, 0
    img_tokenizer_num_tokens = N_IMG
    max_inference_batch_size = 64


class StandIn:
    """Prefill: one image code (context length + 7) to draw, K|V entries equal to the context length.  chunk_run:
    records its inputs, appends n tokens, and leaves code 500 + call index to draw.  generate_run: 1000 * row + step."""

    def __init__(self, vocab, maxlen=400):
        self.V = vocab
        self.transformer = types.SimpleNamespace(mems_mode='kv', hidden_size=H, layers=[None] * L,
                                                 max_memory_length=maxlen,
                                                 position_embeddings=types.SimpleNamespace(weight=torch.zeros(1)))
        self.prefills, self.chunks, self.runs = [], [], []

    def __call__(self, tokens, position_ids, attention_mask, txt, img, is_sparse, *mems):
        assert not mems and tokens.shape[0] == 1 and is_sparse == 0
        C = tokens.shape[1]
        self.prefills.append((tokens.clone(), position_ids.clone()))
        logits = torch.full((1, C, self.V), -1e4)
        logits[0, -1, C + 7] = 0.0
        kv = [torch.full((1, C, 2 * H), float(C), dtype=torch.bfloat16) for _ in range(L)]
        return (logits, *kv, torch.empty((1, C, 0)))

    def _grow(self, mems, n):
        b, t = mems[0].shape[:2]
        return [torch.zeros((b, t + n, 2 * H), dtype=torch.bfloat16) for _ in range(L)] + [torch.empty((b, t + n, 0))]

    def chunk_run(self, tokens, position_ids, mems, row_pad=None):
        assert row_pad is not None and tokens.shape == position_ids.shape
        self.chunks.append(dict(tokens=tokens.clone(), pos=position_ids.clone(), t=mems[0].shape[1],
                                row_pad=row_pad.tolist()))
        logits = torch.full((tokens.shape[0], self.V), -1e4)
        logits[:, 500 + len(self.chunks)] = 0.0
        return logits, self._grow(mems, tokens.shape[1])

    def generate_run(self, last_tokens, first_pos, mems, n_steps, temperature, top_k, invalid_slices, sparse=None,
                     row_pad=None):
        assert sparse is None and row_pad is not None
        b = last_tokens.shape[0]
        self.runs.append(dict(last=last_tokens.clone().view(-1).tolist(), first_pos=[int(p) for p in first_pos],
                              t=mems[0].shape[1], n_steps=n_steps, invalid=[(s.start, s.stop) for s in invalid_slices]))
        new = torch.arange(b).unsqueeze(1) * 1000 + torch.arange(n_steps).unsqueeze(0)
        return new, torch.zeros(b), self._grow(mems, n_steps)


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=N_IMG, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def _interleaved(tok, n_text, given, seed=0, roi2_at=None, nb=1):
    """[ROI1] text [BASE] [BOI2] then: generate 3, given `given[0]` codes, generate 4, given `given[1]`, generate 2."""
    g = torch.Generator().manual_seed(seed)
    text = (N_IMG + torch.randint(0, N_TXT, (n_text,), generator=g)).tolist()
    ctx = [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI2]']]
    if roi2_at is not None:
        ctx[roi2_at] = tok['[ROI2]']
    tail = [-nb] * 3 + given[0] + [-nb] * 4 + given[1] + [-nb] * 2
    return torch.tensor(ctx + tail)


def test_interleaved_templates_share_one_batch(tok):
    from cogview_b200.generation import sampling
    seqs = [_interleaved(tok, n, [[10 + n] * 5, [20 + n] * 2], seed=n) for n in (4, 9, 30)]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        out = sampling.filling_sequences(m, seqs, _Args)
    ctx = [n + 3 for n in (4, 9, 30)]
    T = max(ctx)
    assert len(m.prefills) == 3 and len(m.chunks) == 2 and len(m.runs) == 3
    # stretch 0: first draw from the prefill, then 2 generated; stretch 1: chunk of last + 5 given, then 3 generated
    assert [r['n_steps'] for r in m.runs] == [2, 3, 1]
    assert m.runs[0]['last'] == [C + 7 for C in ctx] and m.runs[0]['t'] == T
    assert m.chunks[0]['t'] == T + 2 and m.chunks[0]['row_pad'] == [T - C for C in ctx]
    assert m.chunks[0]['tokens'][:, 1:].tolist() == [[10 + n] * 5 for n in (4, 9, 30)]
    assert m.chunks[0]['tokens'][:, 0].tolist() == [1000 * r + 1 for r in range(3)]     # the pending token
    assert m.chunks[1]['t'] == T + 2 + 6 + 3 and m.chunks[1]['tokens'].shape == (3, 3)
    assert m.runs[1]['last'] == [501] * 3 and m.runs[2]['last'] == [502] * 3
    for r, (o, seq, C) in enumerate(zip(out, seqs, ctx)):
        assert o.shape == (1, len(seq))
        row = o[0].tolist()
        want = seq.tolist()[:C] + [C + 7, 1000 * r, 1000 * r + 1] + seq.tolist()[C + 3:C + 8] \
            + [501] + [1000 * r + i for i in range(3)] + seq.tolist()[C + 12:C + 14] + [502, 1000 * r]
        assert row == want


def test_rows_keep_their_own_roi2_offsets(tok):
    """Positions after a row's [ROI2] restart from it: each chunk and each generate run gets per-row positions."""
    from cogview_b200.generation import sampling
    seqs = [_interleaved(tok, 6, [[1] * 5, [2] * 2], roi2_at=4), _interleaved(tok, 12, [[1] * 5, [2] * 2], roi2_at=9),
            _interleaved(tok, 8, [[1] * 5, [2] * 2])]
    ctx, offs = [9, 15, 11], [4, 9, 100000]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        sampling.filling_sequences(m, seqs, _Args)

    def p(a, o):
        return a - o if a > o else a
    for (_, pos), C, o in zip(m.prefills, ctx, offs):
        assert pos[0].tolist() == [p(a, o) for a in range(C)]
    assert m.runs[0]['first_pos'] == [p(C, o) for C, o in zip(ctx, offs)]
    assert m.chunks[0]['pos'].tolist() == [[p(C + 2 + i, o) for i in range(6)] for C, o in zip(ctx, offs)]
    assert m.runs[1]['first_pos'] == [p(C + 8, o) for C, o in zip(ctx, offs)]
    assert m.chunks[1]['pos'].tolist() == [[p(C + 11 + i, o) for i in range(3)] for C, o in zip(ctx, offs)]


def test_a_given_roi2_moves_the_offset_of_its_row(tok):
    from cogview_b200.generation import sampling
    r2 = tok['[ROI2]']
    seqs = [_interleaved(tok, 6, [[1, 1, r2, 1, 1], [2, 2]]), _interleaved(tok, 10, [[1] * 5, [2, 2]])]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        sampling.filling_sequences(m, seqs, _Args)
    C0, C1 = 9, 13
    roi = C0 + 3 + 2                                         # absolute position of the given [ROI2] of row 0
    assert m.chunks[0]['pos'][0].tolist() == [a - roi if a > roi else a for a in range(C0 + 2, C0 + 8)]
    assert m.chunks[0]['pos'][1].tolist() == list(range(C1 + 2, C1 + 8))
    assert m.runs[1]['first_pos'] == [C0 + 8 - roi, C1 + 8]


def test_long_given_runs_go_in_pieces(tok):
    from cogview_b200 import ops
    from cogview_b200.generation import sampling
    seqs = [_interleaved(tok, n, [[7] * 100, [8]], seed=n) for n in (3, 5)]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        sampling.filling_sequences(m, seqs, _Args)
    assert [c['tokens'].shape[1] for c in m.chunks] == [ops.ATTN_CHUNK_MAX, 101 - ops.ATTN_CHUNK_MAX, 2]
    assert m.chunks[1]['t'] == m.chunks[0]['t'] + ops.ATTN_CHUNK_MAX


def _fallback_calls(monkeypatch, m, seqs, args):
    from cogview_b200.generation import sampling
    calls = []

    def fake(model, seq, a, **kw):
        calls.append(seq.clone())
        return seq.clamp_min(0).unsqueeze(0)
    monkeypatch.setattr(sampling, "filling_sequence", fake)
    with torch.no_grad():
        out = sampling.filling_sequences(m, seqs, args)
    assert len(out) == len(seqs)
    return calls


@pytest.mark.parametrize("case", ["top_p", "fast_off", "graph_off", "sparse", "too_many_rows", "structure",
                                  "given_length", "beams", "slices", "no_chunk_run", "too_long", "hidden_mems"])
def test_interleaved_templates_that_cannot_share_a_batch(tok, monkeypatch, case):
    args = type("A", (_Args,), {})
    seqs = [_interleaved(tok, n, [[5] * 5, [6] * 2], seed=n) for n in (4, 9)]
    m = StandIn(tok.num_tokens)
    if case == "top_p":
        args.top_p = 0.9
    elif case == "fast_off":
        monkeypatch.setenv("COGVIEW_B200_FAST_DECODE", "0")
    elif case == "graph_off":
        monkeypatch.setenv("COGVIEW_B200_GRAPH_SAMPLING", "0")
    elif case == "sparse":
        args.is_sparse = 2
    elif case == "too_many_rows":
        seqs = [_interleaved(tok, 4, [[5] * 5, [6] * 2], seed=i) for i in range(65)]
    elif case == "structure":
        seqs[1] = torch.cat((seqs[1], torch.tensor([-1])))
    elif case == "given_length":
        seqs[1] = _interleaved(tok, 9, [[5] * 4, [6] * 3])
    elif case == "beams":
        seqs = [_interleaved(tok, n, [[5] * 5, [6] * 2], seed=n, nb=2) for n in (4, 9)]
    elif case == "slices":
        seqs[1] = _interleaved(tok, 9, [[5] * 4 + [tok['[EOI1]']], [6] * 2])
    elif case == "no_chunk_run":
        m = types.SimpleNamespace(**{k: getattr(m, k) for k in ('transformer', 'generate_run')})
    elif case == "too_long":
        m.transformer.max_memory_length = 26                 # longest context 12 + 16 slots after it - 1 > 26
    elif case == "hidden_mems":
        m.transformer.mems_mode = 'hidden'
    calls = _fallback_calls(monkeypatch, m, seqs, args)
    assert len(calls) == len(seqs) and all(torch.equal(c, s) for c, s in zip(calls, seqs))
    if hasattr(m, 'chunks'):
        assert not m.chunks and not m.runs and not m.prefills


def test_single_stretch_templates_keep_their_path(tok):
    """A context followed by one generate run goes through the one-run batch as before, never through chunk_run."""
    from cogview_b200.generation import sampling
    seqs = [torch.tensor([tok['[ROI1]']] + [N_IMG + 1] * n + [tok['[BASE]'], tok['[BOI1]']] + [-1] * 6)
            for n in (3, 8)]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        sampling.filling_sequences(m, seqs, _Args)
    assert not m.chunks and len(m.runs) == 1 and m.runs[0]['n_steps'] == 5


def test_magnify_batch_builds_the_templates_magnify_builds(tok):
    """With a stand-in fill that records every template and fills slot j of a template with a value derived from the
    template itself, magnify_batch gives the same window templates and the same 64 x 64 grids as N magnify calls."""
    from cogview_b200.generation import magnify as mg

    def fill_one(seq):
        out = seq.clone()
        gen = (out < 0).nonzero().view(-1)
        out[gen] = (seq.clamp_min(0).sum() + gen * 7) % N_IMG
        return out.unsqueeze(0)

    solo_tmpls, batch_tmpls = [], []

    def solo_fill(model, seq, args, **kw):
        solo_tmpls.append(seq.clone())
        return fill_one(seq)

    def batch_fill(model, seqs, args):
        batch_tmpls.append([s.clone() for s in seqs])
        return [fill_one(s) for s in seqs]

    g = torch.Generator().manual_seed(3)
    n = 3
    codes = torch.randint(0, N_IMG, (n, 1024), generator=g)
    texts = [torch.tensor([tok['[ROI1]']] + (N_IMG + torch.randint(0, N_TXT, (k,), generator=g)).tolist()
                          + [tok['[BASE]'], tok['[BOI1]']]) for k in (2, 7, 19)]
    solo = torch.cat([mg.magnify(None, tok, codes[r], texts[r], _Args, fill=solo_fill) for r in range(n)])
    batch = mg.magnify_batch(None, tok, codes, texts, _Args, fill=batch_fill)
    assert batch.shape == (n, 4096) and torch.equal(batch, solo)
    assert len(batch_tmpls) == len(mg.WINDOWS)
    for w in range(len(mg.WINDOWS)):
        for r in range(n):
            assert torch.equal(batch_tmpls[w][r], solo_tmpls[r * len(mg.WINDOWS) + w])


def test_super_resolution_batch_groups_and_single_images(tok, monkeypatch):
    from cogview_b200 import generate
    calls = []

    def fake_magnify_batch(model, tokenizer, codes, texts, args, fill=None):
        calls.append(('batch', codes.shape[0]))
        return codes.repeat(1, 4)

    def fake_magnify(model, tokenizer, tokens_list, text, args, fill=None):
        calls.append(('solo', 1))
        return tokens_list.repeat(4).view(1, -1)
    monkeypatch.setattr(generate, "magnify_batch", fake_magnify_batch)
    monkeypatch.setattr(generate, "magnify", fake_magnify)
    args = type("A", (_Args,), {"max_inference_batch_size": 4})
    seqs = [torch.cat((torch.tensor([tok['[ROI1]'], N_IMG + 1, tok['[BASE]'], tok['[BOI1]']]),
                       torch.full((1024,), i))) for i in range(9)]
    model = types.SimpleNamespace(eval=lambda: None)
    codes, imgs = generate.super_resolution_batch(model, None, args, seqs,
                                                  decode=lambda c: c.float().mean().view(1, 1, 1, 1).expand(1, 3, 2, 2))
    assert calls == [('batch', 4), ('batch', 4), ('solo', 1)]
    assert codes.shape == (9, 4096) and [int(c[0]) for c in codes] == list(range(9))
    assert imgs.shape == (9, 3, 2, 2) and [float(i[0, 0, 0]) for i in imgs] == [float(i) for i in range(9)]
