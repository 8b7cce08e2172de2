"""GPU tests of completing partly given images in one decode batch: the forced slots of the graph-replayed decode
(GPT2Model.generate_run with `forced`), filling_completions against filling_sequence per template, and
generate.complete_images end to end with the real-shaped VQ-VAE.

Tolerances (those of test_sr_batch_gpu.py): a teacher-forced run's K|V cache and last-step logits against one prefill
of the whole row through GPT2Model.forward, to 2e-2 of the scale (the abs-max LayerNorm scales of the decode step are
taken over the whole batch); greedy tokens equal a template's solo run up to the first generated slot whose solo
top-2 logit margin is within 2e-2 of the logit scale; sampled tokens lie in the nucleus of a teacher-forced forward
with the route allowance of test_top_p_gpu.py (logits within d = 1e-2 of the scale, a 1e-5 rounding band).
"""
import math

import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu

N_TXT = 101
CFG_GEN = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=256, num_attention_heads=4)
CFG_4B_WIDTH = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=2560, num_attention_heads=40)
MAXLEN = 1100
BAND = 1e-5


def _model(cfg, seed=31):
    from cogview_b200.model import GPT2Model
    m = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                  num_attention_heads=cfg["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=MAXLEN,
                  max_memory_length=MAXLEN, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(max_sequence_length=MAXLEN, seed=seed, **cfg))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    return m


_MODELS = {}


def _get(name):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    if name not in _MODELS:
        _MODELS.clear()                                 # one model at a time
        _MODELS[name] = _model(CFG_GEN if name == "gen" else CFG_4B_WIDTH)
    return _MODELS[name]


class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 1, 0.0, 0
    img_tokenizer_num_tokens = 8192
    max_inference_batch_size = 64


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def _causal(n):
    return torch.tril(torch.ones((1, 1, n, n), device="cuda"))


def _replays(model, b):
    caches = model.transformer.__dict__.get('_kv_pool', {}).get(b)
    runner = getattr(caches, 'runner', None)
    return 0 if runner is None else runner.replays


# ----------------------------------------------------------------------------------------------------
# 1. every slot forced: the run is a prefill of the whole row
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,lens,S", [("gen", (9, 30, 100), 40), ("gen", (3, 50, 64, 17, 200, 5), 17),
                                         ("gen", tuple(5 + 13 * i for i in range(20)), 9),
                                         ("4b", (20, 300, 77), 24)])
def test_teacher_forced_run_is_a_prefill_of_the_whole_row(name, lens, S):
    from cogview_b200.mpu import kv_cache
    model = _get(name)
    b = len(lens)
    g = torch.Generator().manual_seed(sum(lens) + S)
    rows = [torch.randint(0, 8192, (n + S + 1,), generator=g).cuda() for n in lens]
    with torch.no_grad():
        def prefill(r):
            n = lens[r]
            _, *m = model(rows[r][:n].view(1, -1), torch.arange(n, device="cuda").view(1, -1), _causal(n), None, None,
                          0, logits_last_only=True)
            return m
        mems, row_pad = kv_cache.assemble_rows(model.transformer, list(lens), [1] * b, S, prefill)
        last = torch.stack([r[n:n + 1] for r, n in zip(rows, lens)])
        forced = torch.stack([r[n + 1:n + 1 + S] for r, n in zip(rows, lens)])
        toks, _, bm = model.generate_run(last, list(lens), mems, S, 1.0, 0, [slice(8192, None)], row_pad=row_pad,
                                         forced=forced)
        assert torch.equal(toks, forced)
        step_logits = model.transformer._kv_pool[b].runner.step_logits.clone()
        caches = [x[:, :max(lens) + S].clone() for x in bm[:-1]]
        for r, n in enumerate(lens):
            lg, *ms = model(rows[r][:n + S].view(1, -1), torch.arange(n + S, device="cuda").view(1, -1),
                            _causal(n + S), None, None, 0)
            ls = lg[0, -1].float()
            scale = ls.abs().max().item()
            err = (step_logits[r] - ls).abs().max().item()
            print("%s rows %d, row %d (len %d + %d): logits max|diff| %.3e (scale %.3e)" % (name, b, r, n, S, err,
                                                                                             scale))
            assert err < 2e-2 * scale
            for i in range(len(caches)):
                kb, ks = caches[i][r, n:n + S].float(), ms[i][0, n:n + S].float()
                assert (kb - ks).abs().max().item() < 2e-2 * ks.abs().max().item(), (r, i)


# ----------------------------------------------------------------------------------------------------
# 2.-3. greedy rows follow each template alone; given codes come back unchanged
# ----------------------------------------------------------------------------------------------------
def _masks(n, g):
    """Rectangles, [ImageN] prefixes (the codes after the first N) and scattered codes, in turn."""
    out = []
    for i in range(n):
        kind = i % 3
        if kind == 0:
            i0, j0 = (int(x) for x in torch.randint(0, 28, (2,), generator=g))
            h, w = (int(x) for x in torch.randint(1, 9, (2,), generator=g))
            m = torch.zeros((32, 32), dtype=torch.bool)
            m[i0:i0 + h, j0:j0 + w] = True
        elif kind == 1:
            m = (torch.arange(1024) >= int(torch.randint(600, 1020, (1,), generator=g))).view(32, 32)
        else:
            m = torch.zeros(1024, dtype=torch.bool)
            m[torch.randint(0, 1024, (int(torch.randint(2, 25, (1,), generator=g)),), generator=g)] = True
            m = m.view(32, 32)
        out.append(m)
    return out


def _templates(tok, n_img, seed, nb=1):
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    g = torch.Generator().manual_seed(seed)
    seqs = []
    for i, m in enumerate(_masks(n_img, g)):
        text = (8192 + torch.randint(0, N_TXT, (2 + (7 * i) % 40,), generator=g)).tolist()
        codes = torch.randint(0, 8192, (1024,), generator=g)
        seq = torch.tensor(generate.completion_query(text, codes, m, tok), dtype=torch.long, device="cuda")
        sampling.add_interlacing_beam_marks(seq, nb=nb)
        seqs.append(seq)
    return seqs


def _decisive_prefix(model, row, gen_mask):
    """Length of the leading part of `row` that a greedy run must reproduce: up to the first generated slot whose
    top-2 image-code margin in a teacher-forced forward is within 2e-2 of the logit scale."""
    s = row.shape[0]
    with torch.no_grad():
        lg, *_ = model(row[:-1].view(1, -1), torch.arange(s - 1, device="cuda").view(1, -1), _causal(s - 1), None,
                       None, 0)
    lg = lg[0, :, :8192].float()                                  # position j - 1 predicts slot j
    top = lg.topk(2, dim=-1).values
    bad = ((top[:, 0] - top[:, 1] <= 2e-2 * lg.abs().amax(-1)) & gen_mask[1:]).nonzero()
    return 1 + int(bad[0]) if bad.numel() else s


@pytest.mark.parametrize("name,n_img", [("gen", 3), ("gen", 8), ("gen", 16), ("gen", 64), ("4b", 5), ("4b", 17)])
def test_greedy_rows_follow_each_template_alone(tok, name, n_img):
    from cogview_b200.generation import sampling
    model = _get(name)
    seqs = _templates(tok, n_img, seed=n_img)
    tmpls = [s.tolist() for s in seqs]
    with torch.no_grad():
        plans, S, ok = sampling._completion_plan(model, tmpls, _Args, tok)
        assert ok and not sampling._batch_plan(model, tmpls, _Args, tok)[1]
        before = _replays(model, n_img)
        out = sampling.filling_completions(model, seqs, _Args)
        assert _replays(model, n_img) - before == S               # one graph replay per step for all rows
        solo = [sampling.filling_sequence(model, s, _Args) for s in seqs]
    compared = 0
    for o, s, seq in zip(out, solo, seqs):
        assert o.shape == s.shape == (1, len(seq))
        gen = seq < 0
        assert torch.equal(o[0, ~gen], seq[~gen])                 # every given code, bit for bit
        assert int(o[0, gen].min()) >= 0 and int(o[0, gen].max()) < 8192
        k = _decisive_prefix(model, s[0], gen)
        assert torch.equal(o[0, :k], s[0, :k]), (k, int(gen.nonzero()[0]))
        compared += int(gen[:k].sum())
    print("%s, %d images, S = %d: %d generated tokens compared" % (name, n_img, S, compared))
    assert compared > 0


# ----------------------------------------------------------------------------------------------------
# 4. a full mask is the text-to-image template and takes its route
# ----------------------------------------------------------------------------------------------------
def test_a_full_mask_takes_the_text_to_image_route(tok):
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    model = _get("gen")

    class K(_Args):
        top_k = 200
    g = torch.Generator().manual_seed(5)
    seqs = []
    for n in (5, 17, 40):
        text = (8192 + torch.randint(0, N_TXT, (n,), generator=g)).tolist()
        q = generate.completion_query(text, torch.randint(0, 8192, (1024,), generator=g),
                                      torch.ones((32, 32), dtype=torch.bool), tok)
        assert q == generate.build_query(generate.QUERY_TEMPLATES['text2image'], [text], tok)
        seq = torch.tensor(q, dtype=torch.long, device="cuda")
        sampling.add_interlacing_beam_marks(seq, nb=4)
        seqs.append(seq)
    with torch.no_grad():
        torch.manual_seed(9)
        got = sampling.filling_completions(model, seqs, K)
        torch.manual_seed(9)
        want = sampling.filling_sequences(model, seqs, K)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


# ----------------------------------------------------------------------------------------------------
# 5. nucleus sampling of several rows
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("top_k", [0, 200])
def test_nucleus_draws_stay_in_the_nucleus(tok, top_k):
    from cogview_b200.generation import sampling
    model = _get("gen")
    top_p = 0.9

    class P(_Args):
        pass
    P.top_k, P.top_p = top_k, top_p
    seqs = _templates(tok, 6, seed=50 + top_k, nb=2)
    tmpls = [s.tolist() for s in seqs]
    with torch.no_grad():
        _, S, ok = sampling._completion_plan(model, tmpls, P, tok)
        assert ok
        before = _replays(model, 12)
        torch.manual_seed(top_k)
        out = sampling.filling_completions(model, seqs, P)
        assert _replays(model, 12) - before == S
    checked = 0
    for rows, seq in zip(out, seqs):
        nb, s = rows.shape
        gen = seq < 0
        assert nb == 2 and torch.equal(rows[:, ~gen], seq[~gen].expand(nb, -1))
        with torch.no_grad():
            lg, *_ = model(rows[:, :-1].contiguous(), torch.arange(s - 1, device="cuda").repeat(nb, 1),
                           _causal(s - 1), None, None, 0)
        lg = lg.float()
        for j in gen.nonzero().view(-1).tolist():
            full = lg[:, j - 1]                                   # predicts slot j
            d = 1e-2 * full.abs().max().item()
            x = full[:, :8192].double()
            t = rows[:, j].view(-1, 1)
            assert bool((t < 8192).all())
            lt = x.gather(1, t)
            kth = torch.topk(x, top_k)[0][:, -1:] if top_k > 0 else torch.full_like(lt, -float("inf"))
            w = torch.exp(x - x.amax(1, keepdim=True))
            den = (w * (x >= kth - 2 * d)).sum(1)
            lo = math.exp(-2 * d) * (w * (x > lt + 2 * d)).sum(1) / den
            assert bool((lo <= top_p + BAND).all()), (j, lo.max().item(), d)
            checked += nb
    print("top_k=%d, S = %d: %d drawn tokens in the nucleus" % (top_k, S, checked))
    assert checked > 0


# ----------------------------------------------------------------------------------------------------
# 6. complete_images end to end
# ----------------------------------------------------------------------------------------------------
def test_complete_images_with_the_vqvae(tok):
    from cogview_b200 import generate, vqvae
    model = _get("gen")
    vq = vqvae.new_model()
    vq.load_state_dict(recipes.vqvae_state_dict(seed=0))
    vq = vq.cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(3)
    images = torch.randn((3, 3, 256, 256), generator=g, device="cuda")
    codes = vqvae.img2code(vq, images)
    assert codes.shape == (3, 1024) and codes.dtype == torch.int64
    px = torch.zeros((3, 256, 256), dtype=torch.bool, device="cuda")
    px[0, 40:100, 60:200] = True                                  # a rectangle
    px[1, 128:, :] = True                                         # the bottom half: an [Image512] query
    px[2, ::37, ::53] = True                                      # scattered pixels
    masks = generate.code_mask(px)
    texts = [list(range(8192, 8192 + n)) for n in (4, 11, 7)]

    class K(_Args):
        top_k = 200
    out = generate.complete_images(model, vq, K, texts, codes, masks, num=2)
    assert len(out) == 3
    for (rows, imgs), text, c, m in zip(out, texts, codes, masks):
        assert rows.shape == (2, len(text) + 3 + 1024) and imgs.shape == (2, 3, 256, 256)
        flat = m.view(-1)
        got = rows[:, -1024:]
        assert torch.equal(got[:, ~flat], c[~flat].expand(2, -1))
        assert int(got.min()) >= 0 and int(got.max()) < 8192
        with torch.no_grad():
            assert torch.equal(imgs, torch.cat([vqvae.code2img(vq, r.view(1, 1024)) for r in got]))
