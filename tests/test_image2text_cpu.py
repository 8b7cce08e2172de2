"""Host side of image captioning (image2text) with stand-in models: the query layout, how generate.image2text packs
images into decode batches and reads the captions back, and which route filling_shared_prompts takes (one prompt
forward plus a shared-prefix decode run, or filling_sequences)."""
import types

import pytest
import torch

N_IMG, N_TXT = 8192, 101
H, L = 4, 2


class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 200, 0.0, 0
    img_tokenizer_num_tokens = N_IMG
    max_inference_batch_size = 64


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=N_IMG, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def _query(tok, codes, nb):
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    seq = torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['image2text'], [codes], tok))
    sampling.add_interlacing_beam_marks(seq, nb=nb)
    return seq


def test_query_layout(tok):
    from cogview_b200.generation import sampling
    codes = list(range(3, 1027))
    seq = _query(tok, codes, 8)
    assert seq.shape == (1048,)
    assert seq[:2].tolist() == [tok['[BASE]'], tok['[BOI1]']] and seq[2:1026].tolist() == codes
    assert seq[1026:1028].tolist() == [tok['[EOI1]'], tok['[ROI1]']] and seq[1028:].tolist() == [-8] * 20
    C, offset, inv = sampling._scan_context(seq.tolist(), tok)
    assert C == 1028 and offset == 100000
    assert [(s.start, s.stop) for s in inv] == [(0, N_IMG), (N_IMG + N_TXT, None)]      # text ids only


def test_caption_ids_are_the_text_after_roi1(tok):
    from cogview_b200 import generate
    row = _query(tok, [5] * 1024, 1)
    row[1028:] = N_IMG + torch.arange(20)
    assert generate.caption_ids(row, tok) == list(range(20))
    assert generate.caption_ids(row.tolist(), tok) == list(range(20))


class _Fill:
    """Stand-in `fill`: records the templates of every call and fills the slots with 1000 * call + row."""

    def __init__(self, tok):
        self.calls = []

    def __call__(self, model, seqs, args):
        self.calls.append([s.clone() for s in seqs])
        out = []
        for s in seqs:
            nb = -int(s[-1])
            C = int((s >= 0).sum())
            rows = s.view(1, -1).repeat(nb, 1)
            rows[:, C:] = N_IMG + (len(self.calls) - 1) * 10 + torch.arange(nb).view(-1, 1)
            out.append(rows)
        return out


class _Model:
    def eval(self):
        return self


def _images(n):
    return torch.arange(n, dtype=torch.float32).view(n, 1, 1, 1).expand(n, 3, 256, 256)


def _encode(imgs):
    return imgs[:, 0, :32, :32].reshape(imgs.shape[0], 1024).long() + 1


@pytest.mark.parametrize("n,num,mbz,batches", [(3, 8, 64, [3]), (10, 8, 64, [8, 2]), (5, 4, 8, [2, 2, 1]),
                                               (2, 1, 64, [2]), (2, 16, 8, [1, 1, 1, 1])])
def test_images_are_packed_whole_into_batches(tok, n, num, mbz, batches):
    from cogview_b200 import generate

    class A(_Args):
        max_inference_batch_size = mbz
    fill = _Fill(tok)
    out = generate.image2text(_Model(), None, A, _images(n), num=num, fill=fill, encode=_encode)
    nb = min(num, mbz)
    assert [len(c) for c in fill.calls] == batches
    assert all(len(c) * nb <= mbz for c in fill.calls)
    for c in fill.calls:
        for s in c:
            assert s.shape == (1048,) and s[1028:].tolist() == [-nb] * 20
    assert len(out) == n
    for i, (rows, captions) in enumerate(out):
        assert rows.shape == (num, 1048) and len(captions) == num
        assert rows[:, 2:1026].eq(i + 1).all()                          # the image's own codes
        for row, cap in zip(rows, captions):
            assert cap == (row[1028:] - N_IMG).tolist()


def test_num_must_divide_into_batches(tok):
    from cogview_b200 import generate

    class A(_Args):
        max_inference_batch_size = 8
    with pytest.raises(AssertionError):
        generate.image2text(_Model(), None, A, _images(1), num=12, fill=_Fill(tok), encode=_encode)


class StandIn:
    """The prompt forward at batch N: logits that leave one text id (N_IMG + 3 + image) to draw, K|V stand-ins.
    shared_run: records its arguments and returns 100 + row * 1000 + step."""

    def __init__(self, vocab, hidden=H, maxlen=1100):
        self.V = vocab
        self.transformer = types.SimpleNamespace(mems_mode='kv', hidden_size=hidden, layers=[None] * L,
                                                 max_memory_length=maxlen)
        self.forwards, self.runs = [], []

    def __call__(self, tokens, position_ids, attention_mask, txt, img, is_sparse, *mems, logits_last_only=False):
        assert not mems and is_sparse == 0 and logits_last_only
        N, C = tokens.shape
        self.forwards.append((tokens.clone(), position_ids.clone(), attention_mask.shape))
        logits = torch.full((N, 1, self.V), -1e4)
        logits[torch.arange(N), 0, N_IMG + 3 + torch.arange(N)] = 0.0
        kv = [torch.zeros((N, C, 2 * H), dtype=torch.bfloat16) for _ in range(L)]
        return (logits, *kv, torch.empty((N, C, 0)))

    def generate_run(self, *a, **kw):
        raise AssertionError('the shared route does not use generate_run')

    def shared_run(self, last_tokens, first_pos, mems, n_steps, temperature, top_k, invalid_slices):
        b = last_tokens.shape[0]
        self.runs.append(dict(last=last_tokens.clone(), first_pos=first_pos, groups=mems[0].shape[0],
                              P=mems[0].shape[1], n_steps=n_steps, invalid=[(s.start, s.stop) for s in invalid_slices]))
        return 100 + torch.arange(b).unsqueeze(1) * 1000 + torch.arange(n_steps).unsqueeze(0), torch.zeros(b)


def test_shared_route_runs_one_prompt_forward_and_one_decode_run(tok):
    from cogview_b200.generation import sampling
    nb, n = 4, 3
    seqs = [_query(tok, [i + 1] * 1024, nb) for i in range(n)]
    m = StandIn(tok.num_tokens)
    with torch.no_grad():
        out = sampling.filling_shared_prompts(m, seqs, _Args)
    assert len(m.forwards) == 1 and len(m.runs) == 1
    tokens, pos, mask = m.forwards[0]
    assert tokens.shape == (n, 1028) and torch.equal(tokens, torch.stack([s[:1028] for s in seqs]))
    assert torch.equal(pos[0], torch.arange(1028)) and mask == (1, 1, 1028, 1028)
    run = m.runs[0]
    assert run['groups'] == n and run['P'] == 1028 and run['n_steps'] == 19 and run['first_pos'] == 1028
    assert run['invalid'] == [(0, N_IMG), (N_IMG + N_TXT, None)]
    assert run['last'].view(-1).tolist() == [N_IMG + 3 + i for i in range(n) for _ in range(nb)]
    for i, (o, s) in enumerate(zip(out, seqs)):
        assert o.shape == (nb, 1048) and torch.equal(o[:, :1028], s[:1028].expand(nb, -1))
        assert o[:, 1028].eq(N_IMG + 3 + i).all()
        want = 100 + (i * nb + torch.arange(nb)).view(-1, 1) * 1000 + torch.arange(19).view(1, -1)
        assert torch.equal(o[:, 1029:], want)


def _fallback_cases(tok):
    from cogview_b200.generation import sampling

    class Sparse(_Args):
        is_sparse = 1

    class TopP(_Args):
        top_k, top_p = 0, 0.9
    q = [_query(tok, [i + 1] * 1024, 4) for i in range(3)]
    short = _query(tok, [1] * 1024, 4)
    short = torch.cat((short[:1], short[2:]))                              # another context length
    many = [_query(tok, [i + 1] * 1024, 24) for i in range(3)]             # 72 rows
    wide = [_query(tok, [i + 1] * 1024, 8) for i in range(3)]              # 24 rows at a hidden size of 4096
    return [('is_sparse', q, Sparse, {}, None), ('top_p', q, TopP, {}, None), ('hidden', q, _Args, {}, 'hidden'),
            ('72 rows', many, _Args, {}, None), ('hidden 4096', wide, _Args, {}, 4096),
            ('context lengths', q[:2] + [short], _Args, {}, None),
            ('fast decode off', q, _Args, {'COGVIEW_B200_FAST_DECODE': '0'}, None),
            ('graph sampling off', q, _Args, {'COGVIEW_B200_GRAPH_SAMPLING': '0'}, None)]


def test_fallbacks_go_to_filling_sequences(tok, monkeypatch):
    from cogview_b200.generation import sampling
    for name, seqs, args, env, tweak in _fallback_cases(tok):
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            seen = []
            mp.setattr(sampling, 'filling_sequences', lambda model, s, a: seen.append(len(s)) or ['fallback'])
            m = StandIn(tok.num_tokens, hidden=4096 if tweak == 4096 else H)
            if tweak == 'hidden':
                m.transformer.mems_mode = 'hidden'
            with torch.no_grad():
                out = sampling.filling_shared_prompts(m, seqs, args)
            assert out == ['fallback'] and seen == [len(seqs)] and not m.forwards and not m.runs, name


def test_image2text_defaults_to_the_shared_route(tok):
    import inspect
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    assert inspect.signature(generate.image2text).parameters['fill'].default is sampling.filling_shared_prompts
