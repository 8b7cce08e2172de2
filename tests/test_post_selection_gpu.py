"""GPU tests of batched post-selection: cv_vocab_logprob (csrc/vocab_logprob.cu) against a float64 log_softmax,
GPT2Model.token_logprobs against inverse_prompt_score and the oracle, the memory it keeps (none) and allocates, ragged
caption batches through inverse_prompt_scores, and generate.rerank end to end.

Tolerances: the kernel |diff| <= 1e-3 + 1e-4 |logp| against float64 on the same bf16 operands (fp32 accumulation and
exp only); whole-model scores rtol=1e-3, atol=1e-2 as tests/test_decode_mid_gpu.py compares post-selection scores (the
abs-max LayerNorm scale is one scalar per forward tensor, so padded and mixed groups differ in the last bf16 bits).
"""
import pytest
import torch

from oracle import cogview_oracle as O
from oracle import recipes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


# ----------------------------------------------------------------------------------------------------
# 1. the kernel
# ----------------------------------------------------------------------------------------------------
_W = {}


def _weights(V, K):
    if (V, K) not in _W:
        _W.clear()
        g = torch.Generator(device="cuda").manual_seed(V + K)
        _W[(V, K)] = (torch.randn(V, K, generator=g, device="cuda") * (1.0 / K ** 0.5)).to(torch.bfloat16)
    return _W[(V, K)]


def _targets(M, vb, ve, seed):
    """first and last column of the window, both sides of 256-column tile edges, then random columns"""
    special = [vb, ve - 1, vb + 255, vb + 256, vb + 511, vb + 512, ve - 2, vb + 1]
    special = [t for t in special if vb <= t < ve]
    rnd = torch.randint(vb, ve, (M,), generator=torch.Generator().manual_seed(seed))
    t = torch.tensor((special * (M // len(special) + 1))[:M]) if M <= 8 else rnd
    if M > 8:
        t[:len(special)] = torch.tensor(special)
    if M == 1:
        t[0] = ve - 1
    return t.cuda()


def _want(h, w, t, vb, ve):
    lg = h.double() @ w[vb:ve].double().t()
    lp = torch.log_softmax(lg, dim=-1)
    inside = (t >= vb) & (t < ve)
    out = torch.full((h.shape[0],), -float("inf"), dtype=torch.float64, device=h.device)
    out[inside] = lp[inside].gather(1, (t[inside] - vb).view(-1, 1)).view(-1)
    return out


WINDOWS = {"image-masked": (58240, 8192, 58240), "whole": (58240, 0, 58240), "odd": (4999, 257, 4999)}


@pytest.mark.parametrize("window", list(WINDOWS))
@pytest.mark.parametrize("K", [256, 320, 2560])
@pytest.mark.parametrize("M", [1, 7, 128, 129, 1280])
def test_vocab_logprob_matches_float64(ops, M, K, window):
    V, vb, ve = WINDOWS[window]
    w = _weights(V, K)
    g = torch.Generator(device="cuda").manual_seed(M * 7 + K)
    h = torch.randn(M, K, generator=g, device="cuda").to(torch.bfloat16)
    t = _targets(M, vb, ve, M + K)
    got = ops.vocab_logprob(h, w, t, vb, ve)
    want = _want(h, w, t, vb, ve)
    assert got.dtype == torch.float32 and got.shape == (M,) and bool(torch.isfinite(got).all())
    err = (got.double() - want).abs()
    assert bool((err <= 1e-3 + 1e-4 * want.abs()).all()), err.max().item()


@pytest.mark.parametrize("scale", [16.0, 64.0])
def test_vocab_logprob_large_logits(ops, scale):
    """rows scaled up until the logits span hundreds: the per-tile max keeps every exp in range"""
    V, vb, ve = WINDOWS["image-masked"]
    K, M = 2560, 129
    w = _weights(V, K)
    h = (torch.randn(M, K, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda") * scale)
    h = h.to(torch.bfloat16)
    t = _targets(M, vb, ve, 11)
    t[-1] = vb + int((h[-1].float() @ w[vb:ve].float().t()).argmax())    # the most likely token: logp near 0
    want = _want(h, w, t, vb, ve)
    lg = h[:4].double() @ w[vb:ve].double().t()
    assert (lg.amax(1) - lg.amin(1)).min().item() > 100.0
    got = ops.vocab_logprob(h, w, t, vb, ve)
    err = (got.double() - want).abs()
    assert bool(torch.isfinite(got).all()) and bool((err <= 1e-3 + 1e-4 * want.abs()).all()), err.max().item()


def test_vocab_logprob_target_outside_the_window_and_determinism(ops):
    V, vb, ve = WINDOWS["image-masked"]
    K, M = 2560, 1280
    w = _weights(V, K)
    h = torch.randn(M, K, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda").to(torch.bfloat16)
    t = _targets(M, vb, ve, 3)
    t[5], t[6], t[7] = vb - 1, 0, ve          # image tokens and one past the window: -inf, as the masked softmax
    a = ops.vocab_logprob(h, w, t, vb, ve)
    b = ops.vocab_logprob(h, w, t, vb, ve)
    assert torch.equal(a, b)
    assert a[5].item() == a[6].item() == a[7].item() == -float("inf")
    want = _want(h, w, t, vb, ve)
    keep = torch.isfinite(want)
    assert int(keep.sum()) == M - 3
    assert bool(((a.double() - want)[keep].abs() <= 1e-3 + 1e-4 * want[keep].abs()).all())


def test_vocab_logprob_workspace_and_argument_errors(ops):
    lib = ops.lib()
    assert lib.cv_vocab_logprob_workspace_bytes(1280, 8192, 58240) == (196 * 2 + 1) * 1280 * 4
    assert lib.cv_vocab_logprob_workspace_bytes(0, 0, 10) == 0
    w = _weights(4999, 256)
    h = torch.randn(3, 256, device="cuda").to(torch.bfloat16)
    t = torch.zeros(3, dtype=torch.long, device="cuda")
    ws = torch.empty(64, dtype=torch.float32, device="cuda")
    out = torch.empty(3, dtype=torch.float32, device="cuda")
    rc = lib.cv_vocab_logprob(h.data_ptr(), 256, w.data_ptr(), 256, t.data_ptr(), out.data_ptr(), ws.data_ptr(), 3,
                              256, 10, 10, ops.stream_ptr())
    assert rc < 0 and b"v_begin" in lib.cv_last_error()
    with pytest.raises(AssertionError):
        ops.vocab_logprob(h, w, t, 0, 5000)


# ----------------------------------------------------------------------------------------------------
# 2. the model
# ----------------------------------------------------------------------------------------------------
N_TXT = 101          # 8192 image codes + 101 text pieces + 27 command tokens = 8320


class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 200, 0.0, 0
    img_tokenizer_num_tokens = 8192
    max_inference_batch_size = 32


def _model(vocab, seed=31, maxlen=1089):
    from cogview_b200.model import GPT2Model
    cfg = dict(num_layers=2, vocab_size=vocab, hidden_size=256, num_attention_heads=4, max_sequence_length=maxlen)
    m = GPT2Model(num_layers=2, vocab_size=vocab, hidden_size=256, num_attention_heads=4, embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=maxlen,
                  max_memory_length=maxlen, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(seed=seed, **cfg))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    return m, cfg


@pytest.fixture
def small_tok(monkeypatch):
    from cogview_b200.generation import sampling
    tok = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", tok)
    return tok


def _queries(tok, n, text_len, seed, device="cuda"):
    from cogview_b200 import generate
    g = torch.Generator().manual_seed(seed)
    text = (8192 + torch.randint(0, N_TXT, (text_len,), generator=g)).tolist()
    rows = [generate.build_query(generate.QUERY_TEMPLATES['post-selection'],
                                 [torch.randint(0, 8192, (1024,), generator=g).tolist(), text], tok) for _ in range(n)]
    return torch.tensor(rows, dtype=torch.long, device=device)


def test_token_logprobs_match_inverse_prompt_score_and_the_oracle(ops, small_tok):
    from cogview_b200.generation import sampling
    m, cfg = _model(8192 + N_TXT + 27)
    q = _queries(small_tok, 8, 9, seed=1)
    with torch.no_grad():
        want = sampling.inverse_prompt_score(m, q, _Args)
    got = sampling.inverse_prompt_scores(m, q, _Args)
    print("token_logprobs sums vs inverse_prompt_score: max|diff| %.3e" % (got - want).abs().max().item())
    assert torch.allclose(got, want.float(), rtol=1e-3, atol=1e-2)

    # per token, against the fp32 oracle on the bf16-rounded weights (2 rows: the oracle runs on the CPU)
    b, s = 2, q.shape[1]
    tokens = q[:b]
    pos = torch.arange(s, device="cuda").view(1, -1).expand(b, s)
    mask = torch.tril(torch.ones((1, 1, s, s), device="cuda"))
    idx = (torch.arange(b, device="cuda").view(-1, 1) * s + torch.arange(1027, s - 1, device="cuda")).view(-1)
    with torch.no_grad():
        lp = m.token_logprobs(tokens, pos, mask, idx, tokens.view(-1)[idx + 1], vocab_begin=8192)
    sd = {k: v.to(torch.bfloat16).float() for k, v in recipes.gpt2_state_dict(seed=31, **cfg).items()}
    o_logits, _ = O.gpt2_forward(sd, 4, tokens.cpu(), pos.cpu(), mask.cpu())
    o_logits = o_logits.float()
    o_logits[..., :8192] = -float("inf")
    o_lp = torch.log(torch.softmax(o_logits, dim=-1))[:, 1027:-1].gather(2, tokens.cpu()[:, 1028:].unsqueeze(-1))
    o_lp = o_lp.view(-1)
    finite = torch.isfinite(o_lp)
    assert bool(finite.any()) and bool(torch.isfinite(lp).all())
    scale = o_logits[:, 1027:-1, 8192:].abs().max().item()
    err = (lp.cpu() - o_lp)[finite].abs().max().item()
    print("token_logprobs vs oracle: max|diff| %.3e (logit scale %.3e)" % (err, scale))
    assert err < 4e-2 * scale


def test_token_logprobs_keep_no_memory(ops, small_tok):
    from cogview_b200.generation import sampling
    m, _ = _model(8192 + N_TXT + 27)
    tr = m.transformer
    assert tr.max_memory_length == 1089 and tr.mems_mode == "kv"
    q = _queries(small_tok, 4, 6, seed=2)
    with torch.no_grad():                              # a forward that does fill the pool: batch 1
        m(q[:1], torch.arange(q.shape[1], device="cuda").view(1, -1), torch.tril(torch.ones((1, 1, q.shape[1],
                                                                                               q.shape[1]),
                                                                                              device="cuda")),
          None, None, 0)
    pool = dict(tr.__dict__.get("_kv_pool", {}))
    assert pool
    kv, bufs = tr._kv, {k: v.buf.clone() for k, v in pool.items()}
    sampling.inverse_prompt_scores(m, q, _Args)
    assert tr.__dict__.get("_kv_pool") == pool and tr._kv is kv
    for k, v in pool.items():
        # bit for bit: the slots no forward has written hold whatever the allocator left, NaN patterns included
        assert tr._kv_pool[k] is v and torch.equal(v.buf.view(torch.int16), bufs[k].view(torch.int16))
    with pytest.raises(RuntimeError):
        m.token_logprobs(q, torch.arange(q.shape[1], device="cuda").view(1, -1), 0,
                         torch.tensor([1027], device="cuda"), q[0, 1028:1029], vocab_begin=8192)
    with torch.no_grad(), pytest.raises(NotImplementedError):
        m.token_logprobs(q, torch.arange(q.shape[1], device="cuda").view(1, -1), 0,
                         torch.tensor([1027], device="cuda"), q[0, 1028:1029], vocab_begin=8192, is_sparse=2)


def test_peak_memory_of_32_rows_at_the_full_vocabulary(ops, monkeypatch):
    """b = 32 rows of 1039 tokens, V = 58240: the forward's logits alone would be 32 x 1039 x 58240 fp32 (7.7 GB)"""
    from cogview_b200.generation import sampling
    tok = sampling.TokenLayout(img_tokens=8192)          # 50000 text pieces; the model's vocabulary is 58240
    monkeypatch.setattr(sampling, "_TOKENIZER", tok)
    m, _ = _model(58240, seed=3)
    g = torch.Generator().manual_seed(4)
    text = (8192 + torch.randint(0, 50000, (11,), generator=g)).tolist()
    from cogview_b200 import generate
    q = torch.tensor([generate.build_query(generate.QUERY_TEMPLATES['post-selection'],
                                           [torch.randint(0, 8192, (1024,), generator=g).tolist(), text], tok)
                      for _ in range(32)], device="cuda")
    assert q.shape == (32, 1039)
    sampling.inverse_prompt_scores(m, q[:2], _Args)     # warm-up: lazily built state is not part of the call
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    s = sampling.inverse_prompt_scores(m, q, _Args)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    logits_bytes = 32 * 1039 * 58240 * 4
    print("peak during 32-row scoring: %.1f MB (logits would be %.1f MB)" % (peak / 1e6, logits_bytes / 1e6))
    assert bool(torch.isfinite(s).all()) and peak < logits_bytes / 10


def test_ragged_captions_in_one_batch(ops, small_tok):
    from cogview_b200.generation import sampling
    m, _ = _model(8192 + N_TXT + 27)
    per_caption = [_queries(small_tok, 4, n, seed=10 + n) for n in (3, 9, 17)]
    rows = [r for q in per_caption for r in q.unbind(0)]
    order = torch.randperm(len(rows), generator=torch.Generator().manual_seed(0)).tolist()
    mixed = [rows[i] for i in order]
    A32 = type("A32", (_Args,), {"max_inference_batch_size": 32})
    A8 = type("A8", (_Args,), {"max_inference_batch_size": 8})
    got32 = sampling.inverse_prompt_scores(m, mixed, A32)
    got8 = sampling.inverse_prompt_scores(m, mixed, A8)
    alone = torch.cat([sampling.inverse_prompt_scores(m, q, A32) for q in per_caption])[order]
    assert got32.shape == (12,)
    assert torch.allclose(got32, alone, rtol=1e-3, atol=1e-2)
    assert torch.allclose(got8, got32, rtol=1e-3, atol=1e-2)


def test_rerank_end_to_end(ops, small_tok):
    from cogview_b200 import generate, vqvae
    m, _ = _model(8192 + N_TXT + 27)
    vq = vqvae.new_model()
    vq.load_state_dict(recipes.vqvae_state_dict(seed=0))
    vq = vq.cuda().eval()
    A = type("A", (_Args,), {"max_inference_batch_size": 8})
    g = torch.Generator().manual_seed(6)
    seqs = [torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['text2image'],
                                              [(8192 + torch.randint(0, N_TXT, (n,), generator=g)).tolist()],
                                              tokenizer=small_tok), dtype=torch.long, device="cuda") for n in (5, 8)]
    torch.manual_seed(0)
    num, keep = 4, 2
    out = generate.rerank(m, m, vq, A, seqs, num=num, keep=keep)
    assert len(out) == 2
    for seq, r in zip(seqs, out):
        assert r.index.shape == (keep,) and r.rows.shape == (keep, len(seq)) and r.scores.shape == (keep,)
        assert r.images.shape == (keep, 3, 256, 256) and r.all_scores.shape == (num,)
        assert bool(torch.isfinite(r.all_scores).all())
        assert r.index.tolist() == torch.sort(r.all_scores, descending=True, stable=True).indices[:keep].tolist()
        assert torch.equal(r.scores, r.all_scores[r.index])
        assert torch.equal(r.rows[:, :len(seq) - 1024], seq[:-1024].expand(keep, -1))
        with torch.no_grad():
            want = generate._decode_rows(r.rows, lambda c: vqvae.code2img(vq, c))
        assert torch.allclose(r.images, want, atol=1e-5)
        # the scores are the captions' likelihoods of the kept rows
        text = [x + 8192 for x in generate.caption_ids(seq, small_tok)]
        q = generate.post_selection_rows(r.rows, text, small_tok)
        with torch.no_grad():
            again = generate.inverse_prompt_scores(m, q, A)
        assert torch.allclose(again.cpu(), r.scores, rtol=1e-3, atol=1e-2)
