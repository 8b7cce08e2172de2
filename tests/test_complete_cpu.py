"""Host side of completing partly given images in one decode batch, with stand-in models: the completion template
built from codes and masks, code_mask, the decode window filling_completions plans for every row (steps S, window
starts, forced tables, positions, trailing given codes), the templates it hands to filling_sequences, its fallbacks to
filling_sequence per template, and complete_images' batching."""
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
    """Prefill: records its tokens and positions, K|V entries equal to the prompt length.  generate_run: records its
    arguments; a row draws 7000 + row at every step, and a forced token replaces the draw."""

    def __init__(self, vocab, maxlen=1200, hidden=H):
        self.V = vocab
        self.transformer = types.SimpleNamespace(mems_mode='kv', hidden_size=hidden, layers=[None] * L,
                                                 max_memory_length=maxlen,
                                                 position_embeddings=types.SimpleNamespace(weight=torch.zeros(1)))
        self.prefills, self.runs = [], []

    def __call__(self, tokens, position_ids, attention_mask, txt, img, is_sparse, *mems, logits_last_only=False):
        assert not mems and tokens.shape[0] == 1 and is_sparse == 0 and logits_last_only
        C = tokens.shape[1]
        self.prefills.append((tokens.clone(), position_ids.clone()))
        kv = [torch.full((1, C, 2 * H), float(C), dtype=torch.bfloat16) for _ in range(L)]
        return (torch.zeros((1, 1, self.V)), *kv, torch.empty((1, C, 0)))

    def generate_run(self, last_tokens, first_pos, mems, n_steps, temperature, top_k, invalid_slices, sparse=None,
                     row_pad=None, top_p=0.0, forced=None):
        assert sparse is None and row_pad is not None and forced is not None
        b = last_tokens.shape[0]
        self.runs.append(dict(last=last_tokens.view(-1).tolist(), first_pos=[int(p) for p in first_pos],
                              t=mems[0].shape[1], n_steps=n_steps, row_pad=row_pad.tolist(), forced=forced.clone(),
                              invalid=[(s.start, s.stop) for s in invalid_slices], top_p=top_p))
        drawn = (7000 + torch.arange(b)).view(b, 1).expand(b, n_steps)
        new = torch.where(forced >= 0, forced, drawn)
        grown = [torch.zeros((b, mems[0].shape[1] + n_steps, 2 * H), dtype=torch.bfloat16) for _ in range(L)]
        return new, torch.zeros(b), grown + [torch.empty((b, mems[0].shape[1] + n_steps, 0))]


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=N_IMG, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def _text(n, seed):
    return (N_IMG + torch.randint(0, N_TXT, (n,), generator=torch.Generator().manual_seed(seed))).tolist()


def _codes(seed):
    return torch.randint(0, N_IMG, (1024,), generator=torch.Generator().manual_seed(seed))


def _rect(i0, i1, j0, j1):
    m = torch.zeros((32, 32), dtype=torch.bool)
    m[i0:i1, j0:j1] = True
    return m


def _template(tok, n_text, mask, seed=0, nb=1):
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    seq = torch.tensor(generate.completion_query(_text(n_text, seed), _codes(seed), mask, tok))
    sampling.add_interlacing_beam_marks(seq, nb=nb)
    return seq


# ----------------------------------------------------------------------------------------------------
# the template and the code mask
# ----------------------------------------------------------------------------------------------------
def test_completion_query_masks_the_codes(tok):
    from cogview_b200 import generate
    text, codes = _text(7, 1), _codes(1)
    mask = _rect(3, 9, 20, 25)
    mask[31, 31] = True
    q = generate.completion_query(text, codes, mask, tok)
    assert q[:10] == [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']]
    assert len(q) == 10 + 1024
    body = torch.tensor(q[10:])
    flat = mask.view(-1)
    assert bool((body[flat] == -1).all()) and torch.equal(body[~flat], codes[~flat])
    # the same query for a flat mask; nothing masked gives the 'super-resolution' query (the whole image given)
    assert generate.completion_query(text, codes, flat, tok) == q
    assert generate.completion_query(text, codes, torch.zeros(1024, dtype=torch.bool), tok) == generate.build_query(
        generate.QUERY_TEMPLATES['super-resolution'], [text, codes.tolist()], tok)


@pytest.mark.parametrize("n", [0, 1, 333, 1023])
def test_a_mask_of_the_last_codes_is_the_image_n_query(tok, n):
    from cogview_b200 import generate
    text, codes = _text(5, n), _codes(n)
    mask = torch.arange(1024) >= n
    want = generate.build_query('[ROI1] {} [BASE] [BOI1] [Image%d]{}' % n, [text, codes.tolist()], tok)
    assert generate.completion_query(text, codes, mask.view(32, 32), tok) == want


def test_code_mask_takes_any_pixel_of_a_cell():
    from cogview_b200 import generate
    px = torch.zeros((3, 256, 256), dtype=torch.bool)
    px[0, 0, 0] = True                       # one corner pixel: code (0, 0)
    px[1, 15, 255] = True                    # row 15 is in code row 1, column 255 in code column 31
    px[2, 100:140, 8:16] = True              # rows 12..17 of the code grid, column 1
    m = generate.code_mask(px)
    assert m.shape == (3, 32, 32) and m.dtype == torch.bool
    assert m[0].nonzero().tolist() == [[0, 0]]
    assert m[1].nonzero().tolist() == [[1, 31]]
    assert m[2].nonzero().tolist() == [[i, 1] for i in range(12, 18)]
    # against the per-cell loop
    g = torch.Generator().manual_seed(0)
    px = torch.rand((2, 256, 256), generator=g) > 0.9995
    m = generate.code_mask(px)
    for n in range(2):
        for i in range(32):
            for j in range(32):
                assert bool(m[n, i, j]) == bool(px[n, 8 * i:8 * i + 8, 8 * j:8 * j + 8].any())


# ----------------------------------------------------------------------------------------------------
# the plan
# ----------------------------------------------------------------------------------------------------
def _run(tok, seqs, args=_Args, model=None):
    from cogview_b200.generation import sampling
    m = model or StandIn(tok.num_tokens)
    with torch.no_grad():
        out = sampling.filling_completions(m, seqs, args)
    return m, out


def test_rows_of_different_masks_share_one_decode(tok):
    masks = [_rect(4, 8, 10, 20),               # f = C + 138, l = C + 243: 106 slots
             _rect(0, 2, 0, 32),                # f = C, l = C + 63
             torch.arange(1024).view(32, 32) >= 1000,
             _rect(30, 31, 5, 6)]               # one code
    masks[3][31, 0] = True                       # and one more, 27 codes later
    lens = [5, 17, 40, 9]
    seqs = [_template(tok, n, m, seed=i) for i, (n, m) in enumerate(zip(lens, masks))]
    m, out = _run(tok, seqs)
    C = [n + 3 for n in lens]
    f = [C[0] + 138, C[1], C[2] + 1000, C[3] + 965]
    last = [C[0] + 243, C[1] + 63, C[2] + 1023, C[3] + 992]
    S = max(lo - fi + 1 for fi, lo in zip(f, last))
    assert S == 106
    c = [max(2, lo + 1 - S) for lo in last]
    assert all(ci <= fi for ci, fi in zip(c, f)) and c[0] == f[0]
    # one prefill per template, of the tokens before its window; one decode run of S steps
    assert [p[0].shape[1] for p in m.prefills] == [ci - 1 for ci in c]
    assert len(m.runs) == 1
    run = m.runs[0]
    T = max(c) - 1
    assert run['n_steps'] == S and run['t'] == T and run['row_pad'] == [T - (ci - 1) for ci in c]
    assert run['last'] == [s[ci - 1].item() for s, ci in zip(seqs, c)]
    assert run['first_pos'] == [ci - 1 for ci in c]
    assert run['invalid'] == [(N_IMG, None)] and run['top_p'] == 0.0
    for r, (seq, ci) in enumerate(zip(seqs, c)):
        window = seq[ci:ci + S]
        assert torch.equal(run['forced'][r], window.clamp_min(-1))
        # every masked code drawn, every given one (inside the window or after it) unchanged
        o = out[r]
        assert o.shape == (1, len(seq))
        gen = seq < 0
        assert bool((o[0, gen] == 7000 + r).all()) and torch.equal(o[0, ~gen], seq[~gen])
    # row 1's window would start before its second token: it starts there and runs past its last masked code; row
    # 2's starts among the given codes before its masked ones
    assert c[1] == 2 and last[1] + 1 - S < 2 and 2 < c[2] == last[2] + 1 - S < f[2]


def test_a_window_longer_than_the_tail_of_a_short_row_starts_at_its_second_token(tok):
    """Row 1's masked codes end 100 codes in, but row 0 needs 1024 steps: row 1's window starts at slot 2 and
    covers given codes after its last masked one, which are forced."""
    seqs = [_template(tok, 4, torch.ones((32, 32), dtype=torch.bool), seed=1),
            _template(tok, 6, torch.arange(1024).view(32, 32) < 100, seed=2),
            _template(tok, 8, torch.ones((32, 32), dtype=torch.bool), seed=3, nb=1)]
    seqs[2][-1] = 5                                     # the last code given: not the text-to-image layout
    m, out = _run(tok, seqs)
    run = m.runs[0]
    assert run['n_steps'] == 1024
    assert [p[0].shape[1] for p in m.prefills] == [6, 1, 9]
    assert run['forced'][1].tolist() == seqs[1][2:2 + 1024].clamp_min(-1).tolist()
    assert torch.equal(out[1][0, :9], seqs[1][:9]) and bool((out[1][0, 9:109] == 7001).all())
    assert torch.equal(out[1][0, 109:], seqs[1][109:])
    assert out[2][0, -1].item() == 5


def test_beams_share_their_template_prefill(tok):
    seqs = [_template(tok, 5, _rect(2, 4, 0, 8), seed=1, nb=3), _template(tok, 9, _rect(7, 8, 3, 30), seed=2, nb=3)]
    m, out = _run(tok, seqs)
    assert len(m.prefills) == 2 and len(m.runs) == 1
    run = m.runs[0]
    assert len(run['last']) == 6 and run['row_pad'][:3] == [run['row_pad'][0]] * 3
    assert torch.equal(run['forced'][0], run['forced'][2]) and not torch.equal(run['forced'][0], run['forced'][3])
    for i, (o, seq) in enumerate(zip(out, seqs)):
        assert o.shape == (3, len(seq))
        gen = seq < 0
        for b in range(3):
            assert bool((o[b, gen] == 7000 + 3 * i + b).all()) and torch.equal(o[b, ~gen], seq[~gen])


def test_nucleus_sampling_of_several_rows_takes_the_new_route(tok):
    args = type("A", (_Args,), dict(top_p=0.9))
    seqs = [_template(tok, 5, _rect(2, 4, 0, 8), seed=1), _template(tok, 9, _rect(7, 9, 3, 30), seed=2)]
    m, _ = _run(tok, seqs, args)
    assert len(m.runs) == 1 and m.runs[0]['top_p'] == 0.9


def test_a_roi2_before_the_window_restarts_the_positions(tok):
    seqs = [_template(tok, 12, _rect(0, 1, 0, 4), seed=1), _template(tok, 5, _rect(0, 1, 0, 9), seed=2)]
    seqs[0][4] = tok['[ROI2]']
    m, _ = _run(tok, seqs)
    c0 = 15 + 3 + 1 - 9                                  # l = C + 3, S = 9
    assert m.prefills[0][1][0].tolist() == [a - 4 if a > 4 else a for a in range(c0 - 1)]
    assert m.runs[0]['first_pos'][0] == c0 - 1 - 4


# ----------------------------------------------------------------------------------------------------
# the templates filling_sequences batches, and the fallbacks
# ----------------------------------------------------------------------------------------------------
def _spy(monkeypatch):
    from cogview_b200.generation import sampling
    calls = dict(sequences=0, sequence=[])

    def seqs_fake(model, seqs, args):
        calls['sequences'] += 1
        return [s.clamp_min(0).unsqueeze(0) for s in seqs]

    def one_fake(model, seq, args, **kw):
        calls['sequence'].append(seq.clone())
        return seq.clamp_min(0).unsqueeze(0)
    monkeypatch.setattr(sampling, "filling_sequences", seqs_fake)
    monkeypatch.setattr(sampling, "filling_sequence", one_fake)
    return calls


@pytest.mark.parametrize("layout", ["full", "rows", "rect_one_beam"])
def test_templates_of_one_layout_go_to_filling_sequences(tok, monkeypatch, layout):
    """A full mask is the text-to-image template (one generate run); a mask of the last rows is an [ImageN] template;
    the same rectangle in every image with one beam is the interleaved layout of _stretch_plan."""
    from cogview_b200.generation import sampling
    mask = {"full": torch.ones((32, 32), dtype=torch.bool), "rows": torch.arange(1024).view(32, 32) >= 512,
            "rect_one_beam": _rect(3, 9, 4, 20)}[layout]
    seqs = [_template(tok, n, mask, seed=n, nb=4 if layout != "rect_one_beam" else 1) for n in (4, 9, 30)]
    tmpls = [s.tolist() for s in seqs]
    m = StandIn(tok.num_tokens)
    m.chunk_run = lambda *a, **kw: None
    with torch.no_grad():
        assert sampling._batch_plan(m, tmpls, _Args, tok)[1] or sampling._stretch_plan(m, tmpls, _Args, tok)[1]
    calls = _spy(monkeypatch)
    _run(tok, seqs, model=m)
    assert calls['sequences'] == 1 and not calls['sequence'] and not m.runs


@pytest.mark.parametrize("case", ["sparse", "too_many_rows", "hidden", "fast_off", "graph_off", "one_row_top_p",
                                  "no_generate_slot", "beams_differ", "slices", "roi2_in_window", "too_long",
                                  "hidden_mems"])
def test_templates_the_route_refuses_are_filled_one_by_one(tok, monkeypatch, case):
    args = type("A", (_Args,), {})
    seqs = [_template(tok, 5, _rect(2, 4, 0, 8), seed=1), _template(tok, 9, _rect(7, 9, 3, 30), seed=2)]
    m = StandIn(tok.num_tokens)
    if case == "sparse":
        args.is_sparse = 2
    elif case == "too_many_rows":
        seqs = [_template(tok, 5, _rect(2, 4, 0, 8), seed=1, nb=33), _template(tok, 9, _rect(7, 9, 3, 30), seed=2,
                                                                               nb=32)]
    elif case == "hidden":
        m = StandIn(tok.num_tokens, hidden=4096)                # 17..64 rows need a hidden size <= 2560
        seqs = [_template(tok, 5, _rect(2, 4, 0, 8), seed=1, nb=9), _template(tok, 9, _rect(7, 9, 3, 30), seed=2,
                                                                              nb=9)]
    elif case == "fast_off":
        monkeypatch.setenv("COGVIEW_B200_FAST_DECODE", "0")
    elif case == "graph_off":
        monkeypatch.setenv("COGVIEW_B200_GRAPH_SAMPLING", "0")
    elif case == "one_row_top_p":
        args.top_p = 0.9
        seqs = seqs[:1]
    elif case == "no_generate_slot":
        seqs[1] = seqs[1].clamp_min(0)
    elif case == "beams_differ":
        seqs[1][-1] = -2
    elif case == "slices":
        seqs[1][-1] = tok['[EOI1]']                             # text may follow it
        seqs[1] = torch.cat((seqs[1], torch.tensor([-1])))
    elif case == "roi2_in_window":
        f1 = int((seqs[1] < 0).nonzero()[0])
        seqs[1][f1 - 1] = tok['[ROI2]']
    elif case == "too_long":
        m.transformer.max_memory_length = 290               # longest prefill 238 + 59 steps > 290
    elif case == "hidden_mems":
        m.transformer.mems_mode = 'hidden'
    calls = _spy(monkeypatch)
    _run(tok, seqs, args, model=m)
    assert calls['sequences'] == 0 and not m.runs and not m.prefills
    assert len(calls['sequence']) == len(seqs) and all(torch.equal(c, s) for c, s in zip(calls['sequence'], seqs))


def test_one_row_without_nucleus_sampling_takes_the_new_route(tok):
    m, out = _run(tok, [_template(tok, 5, _rect(2, 4, 0, 8), seed=1)])
    assert len(m.runs) == 1 and len(m.runs[0]['last']) == 1


# ----------------------------------------------------------------------------------------------------
# complete_images
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num,mbz", [(1, 64), (4, 8), (16, 8)])
def test_complete_images_batches_whole_images(tok, num, mbz):
    from cogview_b200 import generate
    n = 5
    texts = [_text(3 + i, i) for i in range(n)]
    codes = torch.stack([_codes(i) for i in range(n)])
    masks = torch.stack([_rect(i, i + 3, 2 * i, 2 * i + 5) for i in range(n)])
    args = type("A", (_Args,), dict(max_inference_batch_size=mbz))
    batches = []

    def fill(model, seqs, a):
        batches.append([s.clone() for s in seqs])
        nb = -int(seqs[0].min())
        return [s.clamp_min(0).view(1, -1).repeat(nb, 1) for s in seqs]

    model = types.SimpleNamespace(eval=lambda: None)
    out = generate.complete_images(model, None, args, texts, codes, masks, num=num, fill=fill,
                                   decode=lambda c: torch.zeros((c.shape[0], 3, 256, 256)) + c[:, :1].view(-1, 1, 1, 1))
    nb = min(num, mbz)
    per = max(1, mbz // nb)
    assert [len(b) for b in batches] == [min(per, n - g0) for g0 in range(0, n, per) for _ in range(max(num // mbz, 1))]
    assert all(sum(-int(s.min()) for s in b) <= mbz for b in batches)
    assert len(out) == n
    for i, (rows, imgs) in enumerate(out):
        seq = torch.tensor(generate.completion_query(texts[i], codes[i], masks[i], tok))
        assert rows.shape == (num, len(seq)) and imgs.shape == (num, 3, 256, 256)
        assert torch.equal(rows[:, seq >= 0], seq[seq >= 0].expand(num, -1))
        assert bool((imgs[:, :, 0, 0] == float(rows[0, -1024])).all())      # the decode got the row's codes
