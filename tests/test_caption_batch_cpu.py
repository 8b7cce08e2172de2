"""Host side of sampling many captions in one decode batch, with a stand-in model: which template lists
filling_sequences runs as one ragged batch and which it fills one by one, the batch cache kv_cache.assemble builds
(row_pad, per-row first positions, [ROI2] offsets), the unpacking back to one tensor per caption, and how
generate_images_batch groups captions by max_inference_batch_size and num."""
import types

import pytest
import torch

N_IMG, N_TXT = 8192, 101
H, L = 4, 2


def _tok():
    from cogview_b200.generation import sampling
    return sampling.TokenLayout(img_tokens=N_IMG, txt_tokens=N_TXT)


class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 200, 0.0, 0
    img_tokenizer_num_tokens = N_IMG
    max_inference_batch_size = 64


class StandIn:
    """Prefill: logits that leave one image code (context length + 7) to draw, K|V entries equal to the context
    length.  generate_run: checks the assembled cache and returns 1000 * row + step."""

    def __init__(self, vocab, maxlen=200):
        self.V = vocab
        self.transformer = types.SimpleNamespace(mems_mode='kv', hidden_size=H, layers=[None] * L,
                                                 max_memory_length=maxlen,
                                                 position_embeddings=types.SimpleNamespace(weight=torch.zeros(1)))
        self.prefills, self.runs = [], []

    def __call__(self, tokens, position_ids, attention_mask, txt, img, is_sparse, *mems):
        assert not mems and tokens.shape[0] == 1 and is_sparse == 0
        C = tokens.shape[1]
        self.prefills.append((tokens.clone(), position_ids.clone()))
        logits = torch.full((1, C, self.V), -1e4)
        logits[0, -1, C + 7] = 0.0
        kv = [torch.full((1, C, 2 * H), float(C), dtype=torch.bfloat16) for _ in range(L)]
        return (logits, *kv, torch.empty((1, C, 0)))

    def generate_run(self, last_tokens, first_pos, mems, n_steps, temperature, top_k, invalid_slices, sparse=None,
                     row_pad=None):
        assert sparse is None and row_pad is not None
        b = last_tokens.shape[0]
        t = mems[0].shape[1]
        for i in range(L):
            for r in range(b):
                n = t - int(row_pad[r])
                assert bool((mems[i][r, :n] == n).all())          # the row's own prompt fills slots [0, n)
        self.runs.append(dict(last=last_tokens.clone(), first_pos=list(first_pos), t=t, row_pad=row_pad.tolist(),
                              n_steps=n_steps, invalid=[(s.start, s.stop) for s in invalid_slices]))
        new = torch.arange(b).unsqueeze(1) * 1000 + torch.arange(n_steps).unsqueeze(0)
        return new, torch.zeros(b), mems


def _text2image(tok, n_text, n_gen, nb, seed=0):
    g = torch.Generator().manual_seed(seed)
    text = (N_IMG + torch.randint(0, N_TXT, (n_text,), generator=g)).tolist()
    return torch.tensor([tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + [-nb] * n_gen)


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = _tok()
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def test_captions_of_different_lengths_share_one_ragged_run(tok):
    from cogview_b200.generation import sampling
    nb, n_gen = 4, 10
    seqs = [_text2image(tok, n, n_gen, nb, seed=n) for n in (5, 17, 40)]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        out = sampling.filling_sequences(m, seqs, _Args)
    assert len(m.prefills) == 3 and len(m.runs) == 1
    ctx = [len(s) - n_gen for s in seqs]                           # 8, 20, 43
    for (tokens, pos), C, seq in zip(m.prefills, ctx, seqs):
        assert torch.equal(tokens[0], seq[:C]) and torch.equal(pos[0], torch.arange(C))
    run = m.runs[0]
    assert run['t'] == 43 and run['n_steps'] == n_gen - 1
    assert run['row_pad'] == [43 - C for C in ctx for _ in range(nb)]
    assert run['first_pos'] == [C for C in ctx for _ in range(nb)]
    assert run['last'].view(-1).tolist() == [C + 7 for C in ctx for _ in range(nb)]     # the first draw
    assert run['invalid'] == [(N_IMG, None)]
    for c, (o, seq, C) in enumerate(zip(out, seqs, ctx)):
        assert o.shape == (nb, len(seq))
        assert torch.equal(o[:, :C], seq[:C].expand(nb, -1)) and bool((o[:, C] == C + 7).all())
        rows = torch.arange(c * nb, (c + 1) * nb).unsqueeze(1)
        assert torch.equal(o[:, C + 1:], rows * 1000 + torch.arange(n_gen - 1))


def test_roi2_offsets_give_per_row_first_positions(tok):
    """Low-level super-resolution: positions after [ROI2] restart, so each caption's first generated position is its
    context length minus its own [ROI2] index."""
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    seqs, offsets = [], []
    for n_text in (3, 11):
        text = list(range(N_IMG, N_IMG + n_text))
        q = generate.build_query(generate.QUERY_TEMPLATES['low-level super-resolution'], [text, [5] * 16],
                                 tokenizer=tok)
        q = q[:-1024] + [-1] * 6
        sampling.add_interlacing_beam_marks(q, nb=2)
        seqs.append(torch.tensor(q))
        offsets.append(q.index(tok['[ROI2]']))
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        out = sampling.filling_sequences(m, seqs, _Args)
    ctx = [len(s) - 6 for s in seqs]
    assert m.runs[0]['first_pos'] == [C - o for C, o in zip(ctx, offsets) for _ in range(2)]
    for (tokens, pos), C, o in zip(m.prefills, ctx, offsets):
        want = torch.arange(C)
        want[want > o] -= o
        assert torch.equal(pos[0], want)
    assert [tuple(o.shape) for o in out] == [(2, len(s)) for s in seqs]


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


@pytest.mark.parametrize("case", ["single", "top_p", "fast_off", "graph_off", "too_many_rows", "slot_counts",
                                  "beam_counts", "tokens_after", "sparse", "hidden_mems", "short_run", "too_long"])
def test_templates_that_cannot_share_a_batch_are_filled_one_by_one(tok, monkeypatch, case):
    args = type("A", (_Args,), {})
    seqs = [_text2image(tok, n, 10, 4, seed=n) for n in (5, 17)]
    m = StandIn(tok.num_tokens)
    if case == "single":
        seqs = seqs[:1]
    elif case == "top_p":
        args.top_p = 0.9
    elif case == "fast_off":
        monkeypatch.setenv("COGVIEW_B200_FAST_DECODE", "0")
    elif case == "graph_off":
        monkeypatch.setenv("COGVIEW_B200_GRAPH_SAMPLING", "0")
    elif case == "too_many_rows":
        seqs = [_text2image(tok, n, 10, 33, seed=n) for n in (5, 17)]
    elif case == "slot_counts":
        seqs[1] = _text2image(tok, 17, 11, 4)
    elif case == "beam_counts":
        seqs[1] = _text2image(tok, 17, 10, 2)
    elif case == "tokens_after":
        seqs = [torch.cat((s, torch.tensor([tok['[EOI1]']]))) for s in seqs]
    elif case == "sparse":
        args.is_sparse = 2
    elif case == "hidden_mems":
        m.transformer.mems_mode = 'hidden'
    elif case == "short_run":
        seqs = [_text2image(tok, n, 2, 4, seed=n) for n in (5, 17)]
    elif case == "too_long":
        m.transformer.max_memory_length = 28               # 20 + 9 > 28
    calls = _fallback_calls(monkeypatch, m, seqs, args)
    assert len(calls) == len(seqs) and all(torch.equal(c, s) for c, s in zip(calls, seqs))
    assert not m.runs and not m.prefills


def test_sixty_four_rows_still_share_a_batch(tok):
    from cogview_b200.generation import sampling
    seqs = [_text2image(tok, 10 + 3 * i, 5, 4, seed=i) for i in range(16)]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        out = sampling.filling_sequences(m, seqs, _Args)
    assert len(m.runs) == 1 and m.runs[0]['last'].shape[0] == 64 and len(out) == 16


def test_generate_images_batch_groups_whole_captions(tok):
    from cogview_b200 import generate

    def decode(codes):
        return codes.float().view(1, 1, 32, 32).expand(1, 3, 32, 32) / N_IMG

    groups = []

    def fill(model, seqs, args):
        groups.append([s.clone() for s in seqs])
        out = []
        for s in seqs:
            nb = -int(s[-1])
            row = s.clamp_min(0)
            row[s < 0] = torch.arange(int((s < 0).sum())) % N_IMG
            out.append(row.unsqueeze(0).expand(nb, -1).contiguous())
        return out

    class A(_Args):
        max_inference_batch_size = 8
    seqs = [torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['text2image'], [list(range(N_IMG, N_IMG + n))],
                                              tokenizer=tok)) for n in (4, 9, 2, 7, 5)]
    res = generate.generate_images_batch(torch.nn.Identity(), None, A, seqs, num=4, fill=fill, decode=decode)
    assert [len(g) for g in groups] == [2, 2, 1]
    assert all(bool((s[-1024:] == -4).all()) for g in groups for s in g)      # num beams per caption
    assert len(res) == 5
    for (rows, imgs), seq in zip(res, seqs):
        assert rows.shape == (4, len(seq)) and imgs.shape == (4, 3, 32, 32)
        assert torch.equal(rows[:, :-1024], seq[:-1024].expand(4, -1))
    groups.clear()
    res = generate.generate_images_batch(torch.nn.Identity(), None, A, seqs, num=8, fill=fill, decode=decode)
    assert [len(g) for g in groups] == [1] * 5 and all(r.shape[0] == 8 for r, _ in res)
    groups.clear()
    # more images than one batch holds: generate_images_once per caption, 16 = two fills of 8 beams
    res = generate.generate_images_batch(torch.nn.Identity(), None, A, seqs[:2], num=16, fill=fill, decode=decode)
    assert [len(g) for g in groups] == [1] * 4 and all(bool((g[0][-1024:] == -8).all()) for g in groups)
    assert [tuple(r.shape) for r, _ in res] == [(16, len(s)) for s in seqs[:2]]
    assert [tuple(i.shape) for _, i in res] == [(16, 3, 32, 32)] * 2
