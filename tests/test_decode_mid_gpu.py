"""GPU tests of decoding 17..64 sequences per step: cv_linear_mid_m / cv_ln_pair_mid_m (csrc/decode_mid.cu), the
DecodeRunner built on them, generation with 32 beams and the post-selection driver.

Tolerances: the linear against an fp32 product of the same bf16 inputs — 1e-4 of the row scale for fp32 outputs
(summation order only), 2e-2 for bf16 outputs (rounding of the result); the LayerNorm pair against the 8-row
instance of cv_ln_pair_small_m given the same abs-max scalars — the residual stream y to 1e-6 of its scale, xn to one
bf16 step (same arithmetic, same reduction order) — and against the fp64 oracle; the graph-replayed decode step
against the general GEMM route of GPT2Model.forward — logits within 1e-2 of the logit scale (bf16 paths that differ
in summation order), the appended K|V rows within bf16 rounding, older cache rows untouched.
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


def bf(t):
    return t.to(torch.bfloat16)


def row_err(got, want):
    """max over rows of max|got - want| / max|want| of that row"""
    got, want = got.double().cpu(), want.double().cpu()
    return ((got - want).abs().amax(1) / want.abs().amax(1).clamp_min(1e-30)).max().item()


# ----------------------------------------------------------------------------------------------------
# 1. cv_linear_mid_m
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [17, 24, 33, 63, 64])
@pytest.mark.parametrize("N,K", [(7680, 2560), (2560, 2560), (10240, 2560), (2560, 10240), (58240, 2560), (300, 320)])
def test_linear_mid_m(ops, M, N, K):
    g = torch.Generator().manual_seed(M * 7 + N + K)
    xbuf = torch.zeros((M, K + 8), dtype=torch.bfloat16)
    xbuf[:, :K] = bf(torch.randn((M, K), generator=g))
    xbuf = xbuf.cuda()
    x = xbuf[:, :K]                                              # row stride larger than the row
    w = bf(torch.randn((N, K), generator=g) * 0.05).cuda()
    bias = bf(torch.randn(N, generator=g)).cuda()
    prod = x.float() @ w.float().t()
    guard = 12345.0
    for use_bias, act, dtype in ((True, ops.ACT_NONE, torch.bfloat16), (False, ops.ACT_NONE, torch.float32),
                                 (True, ops.ACT_GELU, torch.bfloat16), (True, ops.ACT_GELU, torch.float32)):
        ref = prod + bias.float() if use_bias else prod
        if act == ops.ACT_GELU:
            ref = O.gelu(ref.double())
        # the output is a window of a larger buffer: one guard row above and below, 16 guard columns to the right
        buf = torch.full((M + 2, N + 16), guard, dtype=dtype, device="cuda")
        out = buf[1:M + 1, :N]
        am = torch.zeros(1, device="cuda")
        ops.linear_mid_m(x, w, bias if use_bias else None, act=act, absmax=am, out=out)
        tag = (use_bias, act, dtype)
        assert row_err(out, ref) < (1e-4 if dtype == torch.float32 else 2e-2), tag
        assert am.item() == out.float().abs().max().item(), tag
        assert bool((buf[0] == guard).all()) and bool((buf[-1] == guard).all()) and bool((buf[:, N:] == guard).all()), tag
        again = torch.empty((M, N), dtype=dtype, device="cuda")
        ops.linear_mid_m(x.contiguous(), w, bias if use_bias else None, act=act, out=again)
        assert torch.equal(again, out), tag                      # same inputs, same bits


def test_linear_mid_m_refuses_other_row_counts(ops):
    from cogview_b200._lib import CogViewB200Error
    w = torch.zeros((64, 64), dtype=torch.bfloat16, device="cuda")
    for M in (16, 65):
        with pytest.raises(CogViewB200Error):
            ops.linear_mid_m(torch.zeros((M, 64), dtype=torch.bfloat16, device="cuda"), w)
        with pytest.raises(CogViewB200Error):
            ops.ln_pair_mid_m(torch.zeros((M, 64), device="cuda"), None, None, None, (w[0], w[0]), 1e-5)


# ----------------------------------------------------------------------------------------------------
# 2. cv_ln_pair_mid_m
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [17, 40, 64])
@pytest.mark.parametrize("K", [320, 2560])
def test_ln_pair_mid_m(ops, M, K):
    g = torch.Generator().manual_seed(M * K + 1)
    res = torch.randn((M, K), generator=g) * (10.0 ** (torch.rand((M, 1), generator=g) * 2 - 1))
    go = bf(torch.randn((M, K), generator=g) * 5)
    gp, bp = bf(1 + 0.1 * torch.randn(K, generator=g)), bf(0.1 * torch.randn(K, generator=g))
    gq, bq = bf(1 + 0.1 * torch.randn(K, generator=g)), bf(0.1 * torch.randn(K, generator=g))
    y_ref = res.double() + O.layernorm_absmax(go.double(), gp.double(), bp.double())
    xn_ref = O.layernorm_absmax(y_ref, gq.double(), bq.double())
    res, go = res.cuda(), go.cuda()
    post, pre = (gp.cuda(), bp.cuda()), (gq.cuda(), bq.cuda())
    am = ops.absmax(go)
    y, xn = ops.ln_pair_mid_m(res, go, am, post, pre, O.LN_EPS)
    assert row_err(y, y_ref) < 1e-4 and row_err(xn, xn_ref) < 2e-2
    _, xn0 = ops.ln_pair_mid_m(res, None, None, None, pre, O.LN_EPS, want_res_out=False)
    assert row_err(xn0, O.layernorm_absmax(res.double().cpu(), gq.double(), bq.double())) < 2e-2
    # The 8-row instance of the small-M kernel has this kernel's thread layout per row.  It takes max|y| over its own 8
    # rows, so every slice is 7 rows of the block plus the row that holds the block's maximum: the same abs-max
    # scalars on both sides, and then the same arithmetic.
    top_y, top_res = int(y.abs().amax(1).argmax()), int(res.abs().amax(1).argmax())
    for r0 in range(0, M, 7):
        rows = [min(r, M - 1) for r in range(r0, r0 + 7)]
        idx = torch.tensor(rows + [top_y], device="cuda")
        ys, xs = ops.ln_pair_small_m(res[idx], go[idx], am, post, pre, O.LN_EPS)
        assert (y[idx] - ys).abs().max().item() <= 1e-6 * ys.abs().max().item(), r0
        assert row_err(xn[idx], xs) < 2.0 ** -7, r0
        idx = torch.tensor(rows + [top_res], device="cuda")
        _, xs0 = ops.ln_pair_small_m(res[idx], None, None, None, pre, O.LN_EPS, want_res_out=False)
        assert row_err(xn0[idx], xs0) < 2.0 ** -7, r0


# ----------------------------------------------------------------------------------------------------
# 3. the decode step
# ----------------------------------------------------------------------------------------------------
CFG_TINY = dict(num_layers=2, vocab_size=58240, hidden_size=256, num_attention_heads=4)
CFG_WIDE = dict(num_layers=2, vocab_size=8192 + 512, hidden_size=2560, num_attention_heads=40)
CFG_MID = dict(num_layers=3, vocab_size=4096, hidden_size=1024, num_attention_heads=16)
CFG_512 = dict(num_layers=2, vocab_size=1000, hidden_size=512, num_attention_heads=8)
CFG_768 = dict(num_layers=2, vocab_size=1000, hidden_size=768, num_attention_heads=12)


def _model(cfg, maxlen, seed=7):
    from cogview_b200.model import GPT2Model
    m = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                  num_attention_heads=cfg["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=maxlen,
                  max_memory_length=maxlen, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"],
                                              hidden_size=cfg["hidden_size"], max_sequence_length=maxlen, seed=seed))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    return m


@pytest.mark.parametrize("cfg,b,t", [(CFG_TINY, 17, 0), (CFG_TINY, 32, 127), (CFG_TINY, 64, 1085), (CFG_TINY, 64, 0),
                                     (CFG_WIDE, 17, 127), (CFG_WIDE, 32, 0), (CFG_WIDE, 32, 1085), (CFG_WIDE, 64, 127),
                                     (CFG_TINY, 1, 0), (CFG_TINY, 3, 17), (CFG_TINY, 4, 120), (CFG_TINY, 8, 64),
                                     (CFG_MID, 2, 33), (CFG_MID, 5, 250), (CFG_512, 4, 40), (CFG_768, 6, 77),
                                     (CFG_WIDE, 4, 0), (CFG_WIDE, 4, 300), (CFG_WIDE, 7, 129), (CFG_WIDE, 8, 1085)])
def test_graph_step_matches_the_general_route(cfg, b, t, monkeypatch):
    """The replayed graph of the decode kernels (the small-M pair up to 16 sequences, the mid-batch pair above)
    against GPT2Model.forward with the fast path switched off (training GEMM tiles, cv_attn_fwd with one query) on
    the same weights and cache."""
    from cogview_b200.mpu import kv_cache
    from cogview_b200.mpu.decode import DecodeRunner
    maxlen = 1089 if t > 200 else 256
    model = _model(cfg, maxlen)
    tr = model.transformer
    g = torch.Generator(device="cuda").manual_seed(100 + b + t)
    c = kv_cache._Caches(tr, b, torch.device("cuda"))
    base = (torch.randn(c.buf.shape, generator=g, device="cuda") * 0.5).to(torch.bfloat16)
    c.buf.copy_(base)
    c.t = t
    r = DecodeRunner(model, c, use_graph=True)
    kind = "small_m" if b <= 16 else "mid_m"
    assert r.linear.__name__ == "linear_" + kind and r.ln_pair.__name__ == "ln_pair_" + kind
    monkeypatch.setenv("COGVIEW_B200_FAST_DECODE", "0")
    mems = [base[i, :, :t].clone() for i in range(cfg["num_layers"])] + [base.new_empty((b, t, 0))] if t > 0 else []
    ids = torch.randint(0, cfg["vocab_size"], (b, 1), generator=torch.Generator().manual_seed(t)).cuda()
    pos = torch.full((b, 1), t, dtype=torch.long, device="cuda")
    with torch.no_grad():
        for step in range(3):
            lp = r.step(ids, pos + step, t + step).clone()
            lo, *mems = model(ids, pos + step, 0, None, None, 0, *mems)
            lo = lo[:, -1].float()
            torch.cuda.synchronize()
            scale = lo.abs().max().item()
            err = (lp - lo).abs().max().item()
            print("h=%d b=%d t=%d step %d: logits max|diff| %.3e (scale %.3e)" % (cfg["hidden_size"], b, t + step, step,
                                                                                 err, scale))
            assert bool(torch.isfinite(lp).all())
            assert err < 1e-2 * scale
            for i in range(cfg["num_layers"]):
                kp, ko = c.buf[i, :, t + step].float(), mems[i][:, t + step].float()
                assert (kp - ko).abs().max().item() < 2e-2 * ko.abs().max().item()
            if t > 0:
                assert torch.equal(c.buf[:, :, :t], base[:, :, :t])
            ids = lo[:, :recipes.IMG_VOCAB].argmax(-1, keepdim=True)
    assert r.replays == 3 and r.graph_launches > 0


def test_mid_batch_step_matches_the_oracle():
    """32 sequences: 16 context tokens through the full forward, then one token through the replayed graph; the fp32
    oracle runs the 17 tokens at once on the bf16-rounded weights."""
    cfg, b, s = CFG_TINY, 32, 16
    model = _model(cfg, 64)
    sd = {k: v.to(torch.bfloat16).float() for k, v in recipes.gpt2_state_dict(
        num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
        max_sequence_length=64, seed=7).items()}
    tokens = torch.randint(0, cfg["vocab_size"], (b, s + 1), generator=torch.Generator().manual_seed(2))
    pos = torch.arange(s + 1).unsqueeze(0).expand(b, s + 1).contiguous()
    with torch.no_grad():
        _, *mems = model(tokens[:, :s].cuda(), pos[:, :s].cuda(), torch.tril(torch.ones((1, 1, s, s), device="cuda")),
                         None, None, 0)
        lg, *mems = model(tokens[:, s:].cuda(), pos[:, s:].cuda(), 0, None, None, 0, *mems)
    runner = model.transformer._kv.runner
    assert runner.replays == 1 and runner.b == b
    o_logits, _ = O.gpt2_forward(sd, cfg["num_attention_heads"], tokens, pos, torch.tril(torch.ones((1, 1, s + 1, s + 1))))
    want = o_logits[:, -1]
    err, scale = (lg[:, -1].float().cpu() - want).abs().max().item(), want.abs().max().item()
    print("b=32 graph step vs oracle: max|diff| %.3e (scale %.3e)" % (err, scale))
    assert err < 2e-2 * scale


# ----------------------------------------------------------------------------------------------------
# 4. generation with 32 beams
# ----------------------------------------------------------------------------------------------------
class _Args:
    temperature, top_p, is_sparse = 1.0, 0.0, 0
    img_tokenizer_num_tokens = recipes.IMG_VOCAB
    max_inference_batch_size = 32


def _fill32(monkeypatch, graph_sampling, top_k, seed, n_gen=40):
    from cogview_b200.generation import sampling
    monkeypatch.setenv("COGVIEW_B200_GRAPH_SAMPLING", "1" if graph_sampling else "0")
    m = _model(CFG_TINY, 128, seed=0)

    class A(_Args):
        pass
    A.top_k = top_k
    tok = sampling.get_tokenizer(A)
    g = torch.Generator().manual_seed(3)
    text = torch.randint(recipes.IMG_VOCAB, recipes.IMG_VOCAB + 100, (18,), generator=g).tolist()
    seq = [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + [-32] * n_gen
    torch.manual_seed(seed)
    with torch.no_grad():
        out = sampling.filling_sequence(m, torch.tensor(seq, dtype=torch.long, device="cuda"), A)
    runner = m.transformer._kv_pool[32].runner
    return out.cpu(), len(seq), runner


def test_filling_sequence_with_32_beams(monkeypatch):
    """top-k = 1 leaves no randomness: the run with the sampling tail inside the replayed graph gives the tokens of
    the per-token host loop over the same step graph.  top-k = 200: valid image codes, beams diverge."""
    eager, n, r_eager = _fill32(monkeypatch, False, 1, 0)
    fused, _, r_fused = _fill32(monkeypatch, True, 1, 0)
    assert eager.shape == fused.shape == (32, n)
    assert torch.equal(eager, fused)
    ngen = n - 21
    # every generated token but the first (it comes from the context's full forward) went through a replayed graph
    assert r_fused.replays >= ngen - 2 and r_eager.replays >= ngen - 2 and r_fused.graph_launches > 0
    assert r_fused.linear.__name__ == "linear_mid_m"
    sampled, _, _ = _fill32(monkeypatch, True, 200, 1)
    gen = sampled[:, 21:]
    assert sampled.shape == (32, n) and int(gen.min()) >= 0 and int(gen.max()) < recipes.IMG_VOCAB
    assert len({tuple(r.tolist()) for r in gen}) > 1


# ----------------------------------------------------------------------------------------------------
# 5. batches of 1..16 are launched as before
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b", [4, 16])
def test_small_batches_keep_their_kernels(ops, b, monkeypatch):
    from cogview_b200.mpu import kv_cache
    from cogview_b200.mpu.decode import DecodeRunner
    model = _model(CFG_TINY, 128)
    counts = []
    for mid_disabled in (False, True):
        if mid_disabled:                                         # no mid-batch range at all: 16 is the only limit
            monkeypatch.setattr(ops, "DECODE_SMALL_MAX_BATCH", 64)
        c = kv_cache._Caches(model.transformer, b, torch.device("cuda"))
        c.buf.zero_()
        c.t = 5
        r = DecodeRunner(model, c, use_graph=True)
        assert r.linear is ops.linear_small_m and r.ln_pair is ops.ln_pair_small_m
        ids = torch.arange(b, device="cuda").view(b, 1) + 5
        with torch.no_grad():
            r.step(ids, torch.full((b, 1), 5, dtype=torch.long, device="cuda"), 5)
        counts.append(r.graph_launches)
    assert counts[0] == counts[1] and counts[0] > 0


# ----------------------------------------------------------------------------------------------------
# 6. draw 32, score them, end to end
# ----------------------------------------------------------------------------------------------------
N_TXT = 101          # small text vocabulary: 8192 image codes + 101 text pieces + 27 command tokens = 8320


def test_generate_32_images_and_post_select(monkeypatch):
    from cogview_b200 import generate, vqvae
    from cogview_b200.generation import sampling
    from cogview_b200.model import GPT2Model
    tok = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", tok)
    cfg = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=256, num_attention_heads=4,
               max_sequence_length=1089)
    m = GPT2Model(num_layers=2, vocab_size=cfg["vocab_size"], hidden_size=256, num_attention_heads=4,
                  embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                  max_sequence_length=1089, max_memory_length=1089, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(seed=31, **cfg))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    vq = vqvae.new_model()
    vq.load_state_dict(recipes.vqvae_state_dict(seed=0))
    vq = vq.cuda().eval()

    class A:
        temperature, top_k, top_p, is_sparse = 1.0, 200, 0.0, 0
        img_tokenizer_num_tokens = 8192
        max_inference_batch_size = 32

    text = (8192 + torch.randint(0, N_TXT, (6,), generator=torch.Generator().manual_seed(4))).tolist()
    seq = torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['text2image'], [text], tokenizer=tok),
                       dtype=torch.long, device="cuda")
    torch.manual_seed(0)
    rows, imgs = generate.generate_images_once(m, vq, A, seq, num=32)
    assert rows.shape == (32, len(seq)) and imgs.shape == (32, 3, 256, 256) and bool(torch.isfinite(imgs).all())
    runner = m.transformer._kv_pool[32].runner
    assert runner.replays >= 1000 and runner.linear.__name__ == "linear_mid_m"
    queries = generate.post_selection_rows(rows, text, tok)
    assert queries.shape == (32, 2 + 1024 + 2 + len(text))
    assert torch.equal(queries[:, 2:1026], rows[:, -1024:]) and bool((queries[:, 1027] == tok['[ROI1]']).all())
    scores = generate.post_selection(m, A, queries)
    assert scores.shape == (32,) and bool(torch.isfinite(scores).all())
    with torch.no_grad():
        one_by_one = torch.cat([sampling.inverse_prompt_score(m, queries[i:i + 1], A) for i in range(32)])
    assert torch.allclose(scores.float(), one_by_one.float(), rtol=1e-3, atol=1e-2)

    A.max_inference_batch_size = 8                                # four groups of eight give the same scores
    assert torch.allclose(generate.post_selection(m, A, queries).float(), scores.float(), rtol=1e-3, atol=1e-2)
