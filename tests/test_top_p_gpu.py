"""GPU tests of nucleus (top-p) sampling: the NUCLEUS instantiation of the fused sampling kernel
(cv_sample_topk with top_p > 0, csrc/sample.cu) and filling_sequence with several beams and top_p > 0 on the
graph-replayed decode path.

* The kernel against a float64 restatement of the rule (top_k_logits, generation/sampling.py:24-49): after the
  temperature, the invalid slices and top-k, a token survives iff the softmax mass of the tokens strictly above it is
  <= top_p.  The kernel adds the mass in 2^-40 fixed point after a float32 exp, so a token whose mass-above lies
  within 1e-5 of top_p (the rounding band) may go either way; every other token must agree.  Ties at the boundary
  are all kept.
* End to end on a 2-layer model: every sampled token lies in the nucleus of the logits of a teacher-forced forward
  over the returned rows.  The decode step and that forward differ by up to d = 1e-2 of the logit scale (the bound of
  test_decode_mid_gpu.py::test_graph_step_matches_the_general_route), which moves each probability by a factor in
  [exp(-2d), exp(2d)] and can swap tokens whose logits lie within 2d.  So a token t is accepted when the mass of the
  tokens whose forward logit exceeds l_t + 2d, times exp(-2d), over the mass of every token the top-k filter of the
  decode step could have kept (forward logit >= k-th largest - 2d), is <= top_p + 1e-5.
"""
import math

import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu

V = 58240
VALID = {"image": [(0, 8192)], "text": [(8192, 58192)], "two": [(0, 8192), (58192, 58240)]}
BAND = 1e-5


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


def _row_logits(b, seed):
    """[b, V] logits whose rows are scaled from 0.3 to 20: nuclei from thousands of tokens down to one."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    scale = torch.exp(torch.linspace(math.log(0.3), math.log(20.0), b, device="cuda")) if b > 1 else \
        torch.full((1,), 3.0, device="cuda")
    return (torch.randn((b, V), generator=g, device="cuda") * scale.view(b, 1)).contiguous()


def _rule(logits, temperature, top_k, top_p, valid):
    """(top-k kept set, mass strictly above every token in float64) of the reference's filters."""
    lg = logits / temperature                                   # the kernel divides in float32 too
    mask = torch.ones_like(lg, dtype=torch.bool)
    for lo, hi in valid:
        mask[:, lo:hi] = False
    lg = lg.masked_fill(mask, -float("inf"))
    if top_k > 0:
        kth = torch.topk(lg, top_k)[0][..., -1, None]
        lg = lg.masked_fill(lg < kth, -float("inf"))
    kept_k = torch.isfinite(lg)
    x = lg.double()
    p = torch.softmax(x, dim=-1)
    neg, order = torch.sort(-x, dim=-1)                         # ascending in -x: descending logits
    ps = p.gather(1, order)
    excl = torch.cumsum(ps, dim=-1) - ps
    first = torch.searchsorted(neg.contiguous(), neg.contiguous(), right=False)   # first index of each tie group
    above_sorted = excl.gather(1, first)
    above = torch.empty_like(above_sorted).scatter_(1, order, above_sorted)
    return kept_k, above


@pytest.mark.parametrize("top_k", [0, 1, 50, 200])
@pytest.mark.parametrize("valid", ["image", "text", "two"])
@pytest.mark.parametrize("b", [1, 5, 64])
def test_kept_set_and_probabilities_match_the_rule(ops, b, valid, top_k):
    rng = VALID[valid]
    logits = _row_logits(b, seed=b * 10 + top_k + len(valid))
    keep = logits.clone()
    banded = checked = 0
    sizes = []
    for temperature in (0.7, 1.0, 1.3):
        for top_p in (1e-6, 0.1, 0.5, 0.9, 0.999):
            nxt, probs = ops.sample_topk(logits, temperature, top_k, rng, seed=17, want_probs=True, top_p=top_p)
            torch.cuda.synchronize()
            assert torch.equal(logits, keep), "the kernel must not modify the logits"
            kept_k, above = _rule(logits, temperature, top_k, top_p, rng)
            want = kept_k & (above <= top_p)
            got = probs > 0
            sure = kept_k & ((above - top_p).abs() > BAND)
            assert torch.equal(got[sure], want[sure]), (temperature, top_p)
            assert not bool((got & ~kept_k).any())
            banded += int((kept_k & ~sure).sum())
            checked += int(sure.sum())
            sizes += got.sum(1).tolist()
            # probabilities: the softmax renormalised over the kept set
            x = (logits / temperature).double().masked_fill(~got, -float("inf"))
            ref = torch.softmax(x, dim=-1)
            assert (probs.double() - ref).abs().max().item() < 1e-6 + 1e-4 * ref.max().item()
            assert bool(got.gather(1, nxt.view(-1, 1)).all())
    print("b=%d %s top_k=%d: %d tokens checked, %d in the rounding band, nucleus sizes %d..%d" % (
        b, valid, top_k, checked, banded, min(sizes), max(sizes)))
    assert min(sizes) >= 1
    if b == 64 and top_k == 0:
        assert min(sizes) == 1 and max(sizes) > 1000


def test_ties_at_the_boundary_are_all_kept(ops):
    logits = torch.full((2, V), -20.0, device="cuda")
    group = [5, 700, 1500, 4000, 8191]                          # spread over the CTA's warps
    logits[:, 3000] = 4.0
    logits[:, group] = 3.0
    logits[:, 6000] = 2.5
    p = torch.softmax(logits[0, :8192].double(), -1)
    p_top, p_tie = p[3000].item(), p[5].item()
    # a sorted cumulative sum crosses top_p at the first, then at the third tied token: the whole group is kept
    for top_p in (p_top + 0.3 * p_tie, p_top + 2.5 * p_tie):
        _, probs = ops.sample_topk(logits, 1.0, 0, [(0, 8192)], seed=1, want_probs=True, top_p=top_p)
        for r in range(2):
            kept = (probs[r] > 0).nonzero().view(-1).tolist()
            assert kept == sorted([3000] + group), (top_p, r, kept)
    # with the whole group above top_p the next token is kept as well
    _, probs = ops.sample_topk(logits, 1.0, 0, [(0, 8192)], seed=1, want_probs=True, top_p=p_top + 5.5 * p_tie)
    assert (probs[0] > 0).nonzero().view(-1).tolist() == sorted([3000, 6000] + group)


@pytest.mark.parametrize("valid", ["image", "text"])
@pytest.mark.parametrize("top_k", [0, 200])
def test_top_p_zero_and_one_match_cv_sample_topk_and_repeats_are_equal(ops, valid, top_k):
    rng = VALID[valid]
    logits = _row_logits(16, seed=3)
    base = ops.sample_topk(logits, 1.0, top_k, rng, seed=99, want_probs=True)
    zero = ops.sample_topk(logits, 1.0, top_k, rng, seed=99, want_probs=True, top_p=0.0)
    one = ops.sample_topk(logits, 1.0, top_k, rng, seed=99, want_probs=True, top_p=1.0)
    for a in (zero, one):
        assert torch.equal(a[0], base[0]) and torch.equal(a[1], base[1])
    reps = [ops.sample_topk(logits, 0.8, top_k, rng, seed=5, want_probs=True, top_p=0.9) for _ in range(3)]
    assert all(torch.equal(r[0], reps[0][0]) and torch.equal(r[1], reps[0][1]) for r in reps[1:])
    assert not torch.equal(reps[0][1] > 0, base[1] > 0)          # the nucleus did cut something


@pytest.mark.parametrize("valid,top_k,top_p,temperature", [("image", 0, 0.9, 1.0), ("image", 200, 0.5, 0.8),
                                                           ("two", 50, 0.9, 1.3), ("text", 0, 0.7, 1.0)])
def test_draws_stay_in_the_nucleus_and_follow_it(ops, valid, top_k, top_p, temperature):
    rng = VALID[valid]
    torch.manual_seed(0)
    b = 4
    logits = (torch.randn((b, V), device="cuda") * 2.5).contiguous()
    _, probs = ops.sample_topk(logits, temperature, top_k, rng, seed=1, want_probs=True, top_p=top_p)
    n = 4000
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.zeros((b, n), dtype=torch.int64, device="cuda")
    score = torch.zeros(b, device="cuda")
    pos = torch.zeros((b, 1), dtype=torch.int64, device="cuda")
    cur = torch.zeros(1, dtype=torch.int32, device="cuda")
    done = torch.zeros(1, dtype=torch.int32, device="cuda")
    ids = torch.zeros(b, dtype=torch.int64, device="cuda")
    seed_dev = torch.tensor([991], dtype=torch.int64, device="cuda")
    for _ in range(n):
        ops.sample_topk(logits, temperature, top_k, rng, seed_dev=seed_dev, step=step, next_ids=ids, out_tokens=out,
                        score_acc=score, pos=pos, cur_len=cur, done=done, top_p=top_p)
    torch.cuda.synchronize()
    assert int(step) == n and int(cur) == n and bool((pos == n).all()) and int(done) == 0
    kept_k, above = _rule(logits, temperature, top_k, top_p, rng)
    nucleus = kept_k & (above <= top_p)
    assert bool(nucleus.gather(1, out).all()), "a draw fell outside the nucleus"
    ref = torch.softmax((logits / temperature).double().masked_fill(~(probs > 0), -float("inf")), dim=-1)
    lp = torch.log(ref.gather(1, out)).sum(1)
    assert torch.allclose(score.double(), lp, rtol=1e-3, atol=1e-2)
    for r in range(b):
        p = ref[r]
        cnt = torch.bincount(out[r], minlength=V).double()
        top = torch.topk(p, 5)
        for pv, iv in zip(top.values.tolist(), top.indices.tolist()):
            sd = math.sqrt(n * pv * (1 - pv)) + 1.0
            assert abs(float(cnt[iv]) - n * pv) < 5 * sd, (r, iv, pv, float(cnt[iv]))


# ----------------------------------------------------------------------------------------------------
# filling_sequence end to end
# ----------------------------------------------------------------------------------------------------
N_TXT = 101
CFG_GEN = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=256, num_attention_heads=4)


def _model(maxlen, seed=31):
    from cogview_b200.model import GPT2Model
    cfg = CFG_GEN
    m = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                  num_attention_heads=cfg["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=maxlen,
                  max_memory_length=maxlen, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"],
                                              hidden_size=cfg["hidden_size"], max_sequence_length=maxlen, seed=seed))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    return m


class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 0, 0.9, 0
    img_tokenizer_num_tokens = 8192
    max_inference_batch_size = 64


@pytest.fixture(scope="module")
def gen_model():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return _model(1100)


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def _template(tok, n_text, nb, n_gen, seed=0):
    g = torch.Generator().manual_seed(seed)
    text = (8192 + torch.randint(0, N_TXT, (n_text,), generator=g)).tolist()
    seq = [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + [-nb] * n_gen
    return torch.tensor(seq, dtype=torch.long, device="cuda")


def _replays(model, nb):
    caches = model.transformer.__dict__.get('_kv_pool', {}).get(nb)
    runner = getattr(caches, 'runner', None)
    return 0 if runner is None else runner.replays


def _fresh_pool(model):
    model.transformer._kv_pool = {}
    model.transformer._kv = None


def _check_nucleus(model, rows, C, top_k, top_p):
    """Every generated token of rows [nb, s] (template slots C ..) lies in the nucleus of the teacher-forced logits,
    within the route tolerance of the module docstring.  Returns (tokens checked, tokens that also pass with d = 0)."""
    nb, s = rows.shape
    with torch.no_grad():
        lg, *_ = model(rows[:, :-1].contiguous(), torch.arange(s - 1, device="cuda").repeat(nb, 1),
                       torch.tril(torch.ones((1, 1, s - 1, s - 1), device="cuda")), None, None, 0)
    lg = lg.float()
    exact = 0
    for j in range(C, s):
        full = lg[:, j - 1]                                       # predicts token j
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
        kept_k = x >= kth
        strict = (w * kept_k * (x > lt)).sum(1) / (w * kept_k).sum(1)
        exact += int((strict <= top_p + BAND).sum())
    return nb * (s - C), exact


@pytest.mark.parametrize("top_k", [0, 200])
@pytest.mark.parametrize("nb", [2, 8, 16, 17, 64])
def test_several_beams_sample_the_nucleus_on_the_graph(gen_model, tok, nb, top_k):
    from cogview_b200.generation import sampling

    class A(_Args):
        pass
    A.top_k = top_k
    seq = _template(tok, 7, nb, 24, seed=nb)
    C = int((seq >= 0).sum())
    before = _replays(gen_model, nb)
    torch.manual_seed(nb)
    with torch.no_grad():
        out = sampling.filling_sequence(gen_model, seq, A)
    assert out.shape == (nb, len(seq)) and torch.equal(out[:, :C], seq[:C].expand(nb, -1))
    assert _replays(gen_model, nb) - before == 23                 # every slot after the first on the graph
    checked, exact = _check_nucleus(gen_model, out, C, top_k, 0.9)
    print("nb=%d top_k=%d: %d tokens in the nucleus, %d of them also without the route tolerance" % (
        nb, top_k, checked, exact))
    assert len({tuple(r.tolist()) for r in out[:, C:]}) > 1


@pytest.mark.parametrize("nb", [8, 17])
def test_tiny_top_p_is_the_arg_max(gen_model, tok, nb):
    from cogview_b200.generation import sampling

    class P(_Args):
        top_k, top_p = 0, 1e-6

    class K(_Args):
        top_k, top_p = 1, 0.0
    seq = _template(tok, 9, nb, 30, seed=1)
    with torch.no_grad():
        torch.manual_seed(2)
        a = sampling.filling_sequence(gen_model, seq, P)
        torch.manual_seed(2)
        b = sampling.filling_sequence(gen_model, seq, K)
    assert torch.equal(a, b)


@pytest.mark.parametrize("switch", ["COGVIEW_B200_FUSED_SAMPLING", "COGVIEW_B200_GRAPH_SAMPLING"])
def test_torch_tail_and_host_loop_sample_the_nucleus(gen_model, tok, monkeypatch, switch):
    from cogview_b200.generation import sampling
    monkeypatch.setenv(switch, "0")
    _fresh_pool(gen_model)                                        # no graph captured with the fused tail
    nb = 8
    seq = _template(tok, 5, nb, 20, seed=4)
    C = int((seq >= 0).sum())
    torch.manual_seed(4)
    with torch.no_grad():
        out = sampling.filling_sequence(gen_model, seq, _Args)
    assert out.shape == (nb, len(seq))
    replays = _replays(gen_model, nb)
    if switch == "COGVIEW_B200_FUSED_SAMPLING":
        assert replays == 19 and gen_model.transformer._kv_pool[nb].runner.sample_graphs
    else:
        assert not gen_model.transformer._kv_pool[nb].runner.sample_graphs    # host loop: decode steps only
    checked, exact = _check_nucleus(gen_model, out, C, 0, 0.9)
    print("%s=0: %d tokens in the nucleus (%d without the route tolerance)" % (switch, checked, exact))
    _fresh_pool(gen_model)


def test_one_row_keeps_the_host_loop(gen_model, tok, monkeypatch):
    from cogview_b200.generation import sampling
    calls = []
    real = gen_model.generate_run

    def spy(*a, **kw):
        calls.append(kw)
        return real(*a, **kw)
    monkeypatch.setattr(gen_model, "generate_run", spy)
    seq = _template(tok, 6, 1, 20, seed=9)
    outs = []
    for _ in range(2):
        torch.manual_seed(21)
        with torch.no_grad():
            outs.append(sampling.filling_sequence(gen_model, seq, _Args))
    assert not calls
    assert outs[0].shape == (1, len(seq)) and torch.equal(outs[0], outs[1])


def test_callers_with_top_p(gen_model, tok):
    """image2text (8 beams per image) and generate_images_batch (4 images per caption) with top_p 0.9."""
    from cogview_b200 import generate

    class A(_Args):
        top_k = 0
    g = torch.Generator().manual_seed(0)

    def encode(imgs):
        return torch.randint(0, 8192, (imgs.shape[0], 1024), generator=g).cuda()
    torch.manual_seed(1)
    out = generate.image2text(gen_model, None, A, torch.zeros((2, 3, 256, 256), device="cuda"), num=8,
                              encode=encode)
    assert len(out) == 2
    for rows, captions in out:
        assert rows.shape == (8, 1048) and len(captions) == 8
        gen = rows[:, 1028:]
        assert int(gen.min()) >= 8192 and int(gen.max()) < 8192 + N_TXT

    def decode(codes):
        return codes.float().view(-1, 1, 32, 32).expand(-1, 3, 32, 32) / 8192
    seqs = [torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['text2image'],
                                              [list(range(8192, 8192 + n))], tokenizer=tok)) for n in (3, 8, 5)]
    res = generate.generate_images_batch(gen_model, None, A, [s.cuda() for s in seqs], num=4, decode=decode)
    assert len(res) == 3
    for (rows, imgs), seq in zip(res, seqs):
        assert rows.shape == (4, len(seq)) and imgs.shape == (4, 3, 32, 32)
        assert int(rows[:, -1024:].min()) >= 0 and int(rows[:, -1024:].max()) < 8192
