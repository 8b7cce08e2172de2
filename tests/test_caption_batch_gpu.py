"""GPU tests of sampling several captions in one decode batch: cv_attn_decode with row_pad (a cache length per row), the
DecodeRunner's ragged mode, and filling_sequences end to end.

Tolerances: the kernel against a float64 softmax over each row's own keys, to one bf16 rounding of the output
(2^-8 relative) plus 1e-3 absolute; a ragged decode step against a step of each caption alone on the same cache
contents, to 1e-2 of the logit scale (the bound of test_decode_mid_gpu.py::test_graph_step_matches_the_general_route:
the abs-max LayerNorm scales are taken over the whole batch, so rows of other captions change them); greedy tokens
equal a caption's solo run up to the first position whose solo top-2 logit margin is within twice that bound (the
margin rule of test_model_gpu.py).
"""
import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu

HD = 64


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


# ----------------------------------------------------------------------------------------------------
# 1. cv_attn_decode with row_pad
# ----------------------------------------------------------------------------------------------------
def _pads(b, cur_len, nsplit, g):
    """Row 0: no pad; row 1: the whole cache (t_b = 0); row 2: more than one split's share; the rest random."""
    pads = torch.randint(0, cur_len + 1, (b,), generator=g)
    pads[0] = 0
    if b > 1:
        pads[1] = cur_len
    if b > 2:
        pads[2] = min(cur_len, cur_len // nsplit + 7)
    return pads.to(torch.int32)


@pytest.mark.parametrize("nsplit", [1, 3, 16])
@pytest.mark.parametrize("heads", [4, 40])
@pytest.mark.parametrize("b", [1, 5, 17, 64])
def test_attn_decode_ragged(ops, b, heads, nsplit):
    h = heads * HD
    for max_len, cur_len in ((1200, 1100), (300, 299), (64, 5)):
        seed = b * 1000 + heads * 10 + nsplit + cur_len
        g, gd = torch.Generator().manual_seed(seed), torch.Generator(device="cuda").manual_seed(seed)
        pads = _pads(b, cur_len, nsplit, g)
        t = (cur_len - pads).tolist()
        cache = torch.randn((b, max_len, 2 * h), generator=gd, device="cuda").to(torch.bfloat16)
        for r in range(b):
            cache[r, t[r]:] = float("nan")                      # never read, never written except slot t_b
        qkv = torch.randn((b, 3 * h), generator=gd, device="cuda").to(torch.bfloat16)
        before = cache.clone()
        cl = torch.tensor([cur_len], dtype=torch.int32, device="cuda")
        out = ops.attn_decode(qkv, cache, heads, cur_len_dev=cl, nsplit=nsplit, row_pad=pads.cuda())
        torch.cuda.synchronize()
        q = qkv[:, :h].double().view(b, heads, HD)
        k_new, v_new = qkv[:, h:2 * h], qkv[:, 2 * h:]
        for r in range(b):
            k = torch.cat((before[r, :t[r], :h], k_new[r:r + 1])).double().view(-1, heads, HD)
            v = torch.cat((before[r, :t[r], h:], v_new[r:r + 1])).double().view(-1, heads, HD)
            p = torch.softmax(torch.einsum("hd,khd->hk", q[r], k) / HD ** 0.5, dim=-1)
            ref = torch.einsum("hk,khd->hd", p, v).reshape(h)
            err = (out[r].double() - ref).abs()
            assert bool((err <= 2.0 ** -8 * ref.abs() + 1e-3).all()), (max_len, cur_len, r, t[r], err.max().item())
            # the append lands at t_b; every other slot of the row keeps its bits (NaN poison included)
            assert torch.equal(cache[r, t[r], :h], k_new[r]) and torch.equal(cache[r, t[r], h:], v_new[r])
            want = before[r].clone()
            want[t[r], :h], want[t[r], h:] = k_new[r], v_new[r]
            assert torch.equal(cache[r].view(torch.int16), want.view(torch.int16)), (r, t[r])
        # all pads zero: the bits of cv_attn_decode at the same nsplit
        base = torch.randn((b, max_len, 2 * h), generator=gd, device="cuda").to(torch.bfloat16)
        c0, c1 = base.clone(), base.clone()
        o0 = ops.attn_decode(qkv, c0, heads, cur_len_dev=cl, nsplit=nsplit)
        o1 = ops.attn_decode(qkv, c1, heads, cur_len_dev=cl, nsplit=nsplit,
                             row_pad=torch.zeros(b, dtype=torch.int32, device="cuda"))
        assert torch.equal(o0, o1) and torch.equal(c0, c1)


# ----------------------------------------------------------------------------------------------------
# 2. the ragged decode step
# ----------------------------------------------------------------------------------------------------
CFG_TINY = dict(num_layers=2, vocab_size=58240, hidden_size=256, num_attention_heads=4)
N_TXT = 101
CFG_GEN = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=256, num_attention_heads=4)


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


@pytest.mark.parametrize("nb,lens", [(4, (9, 30, 100)), (8, (3, 50, 64, 17))])
def test_ragged_step_matches_each_caption_alone(ops, nb, lens):
    from cogview_b200.mpu import kv_cache
    from cogview_b200.mpu.decode import DecodeRunner
    model = _model(CFG_TINY, 256)
    tr = model.transformer
    b, t = nb * len(lens), max(lens)
    g = torch.Generator(device="cuda").manual_seed(b + t)
    c = kv_cache._Caches(tr, b, torch.device("cuda"))
    c.buf.copy_((torch.randn(c.buf.shape, generator=g, device="cuda") * 0.5).to(torch.bfloat16))
    base = c.buf.clone()
    row_len = torch.tensor([n for n in lens for _ in range(nb)])
    row_pad = (t - row_len).to(torch.int32).cuda()
    ids = torch.randint(0, 8192, (b, 1), generator=torch.Generator().manual_seed(1)).cuda()
    pos = row_len.view(b, 1).cuda()
    ragged = DecodeRunner(model, c, use_graph=True)
    c_eager = kv_cache._Caches(tr, b, torch.device("cuda"))
    c_eager.buf.copy_(base)
    eager = DecodeRunner(model, c_eager, use_graph=False)
    solo = []
    for ci, n in enumerate(lens):
        cs = kv_cache._Caches(tr, nb, torch.device("cuda"))
        cs.buf.copy_(base[:, ci * nb:(ci + 1) * nb])
        solo.append((cs, DecodeRunner(model, cs, use_graph=True)))
    with torch.no_grad():
        for step in range(3):
            lg = ragged.step(ids, pos + step, t + step, row_pad=row_pad).clone()
            le = eager.step(ids, pos + step, t + step, row_pad=row_pad).clone()
            assert torch.equal(lg, le)                            # graph replay == per-operation launches
            for ci, n in enumerate(lens):
                rows = slice(ci * nb, (ci + 1) * nb)
                cs, rs = solo[ci]
                ls = rs.step(ids[rows], pos[rows] + step, n + step).clone()
                scale = ls.abs().max().item()
                err = (lg[rows] - ls).abs().max().item()
                print("nb=%d len=%d step %d: logits max|diff| %.3e (scale %.3e)" % (nb, n, step, err, scale))
                assert err < 1e-2 * scale
                for i in range(CFG_TINY["num_layers"]):
                    kp, ko = c.buf[i, rows, n + step].float(), cs.buf[i, :, n + step].float()
                    assert (kp - ko).abs().max().item() < 2e-2 * ko.abs().max().item()
            ids = lg[:, :8192].argmax(-1, keepdim=True)
    assert torch.equal(c.buf, c_eager.buf)
    for ci, n in enumerate(lens):                                 # past every row's end: untouched
        for r in range(ci * nb, (ci + 1) * nb):
            assert torch.equal(c.buf[:, r, n + 3:], base[:, r, n + 3:])


# ----------------------------------------------------------------------------------------------------
# 3.-5. filling_sequences end to end
# ----------------------------------------------------------------------------------------------------
class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 1, 0.0, 0
    img_tokenizer_num_tokens = 8192
    max_inference_batch_size = 64


@pytest.fixture(scope="module")
def gen_model():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return _model(CFG_GEN, 128, seed=31)


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def _captions(tok, text_lens, nb, n_gen, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in text_lens:
        text = (8192 + torch.randint(0, N_TXT, (n,), generator=g)).tolist()
        seq = [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + [-nb] * n_gen
        out.append(torch.tensor(seq, dtype=torch.long, device="cuda"))
    return out


def _decisive_prefix(model, row, C):
    """Number of leading tokens of `row` whose choice had a top-2 margin (image codes, teacher-forced forward) above
    2 x 1e-2 of the logit scale; the context and the first draw (from the context's own forward) always count."""
    s = row.shape[0]
    with torch.no_grad():
        lg, *_ = model(row[:-1].view(1, -1), torch.arange(s - 1, device="cuda").view(1, -1),
                       torch.tril(torch.ones((1, 1, s - 1, s - 1), device="cuda")), None, None, 0)
    lg = lg[0, C:, :8192].float()                                 # predicts tokens C + 1 ..
    top = lg.topk(2, dim=-1).values
    margin = top[:, 0] - top[:, 1]
    bad = (margin <= 2 * 1e-2 * lg.abs().amax(-1)).nonzero()
    return C + 1 + (int(bad[0]) if bad.numel() else s - C - 1)


@pytest.mark.parametrize("n_caps", [3, 8, 16])
def test_greedy_rows_follow_each_caption_alone(gen_model, tok, n_caps):
    from cogview_b200.generation import sampling
    lens = [(5, 17, 40)[i % 3] + i // 3 for i in range(n_caps)]
    seqs = _captions(tok, lens, 4, 48, seed=n_caps)
    with torch.no_grad():
        out = sampling.filling_sequences(gen_model, seqs, _Args)
        solo = [sampling.filling_sequence(gen_model, s, _Args) for s in seqs]
    runner = gen_model.transformer._kv_pool[4 * n_caps].runner
    assert runner.linear.__name__ == ("linear_small_m" if 4 * n_caps <= 16 else "linear_mid_m")
    checked = 0
    for o, s, seq, n in zip(out, solo, seqs, lens):
        assert o.shape == s.shape == (4, len(seq))
        C = n + 3
        k = _decisive_prefix(gen_model, s[0], C)
        assert torch.equal(o[:, :k], s[:, :k]), (n, k)
        checked += k - C
    print("%d captions: %d generated tokens compared" % (n_caps, checked))
    assert checked > 0


def test_top_k_sampling_stays_in_the_image_codes(gen_model, tok):
    from cogview_b200.generation import sampling

    class A(_Args):
        top_k = 200
    seqs = _captions(tok, [5 + 4 * i for i in range(8)], 4, 40, seed=5)
    torch.manual_seed(3)
    with torch.no_grad():
        out = sampling.filling_sequences(gen_model, seqs, A)
    for o, seq in zip(out, seqs):
        C = int((seq >= 0).sum())
        assert o.shape == (4, len(seq)) and torch.equal(o[:, :C], seq[:C].expand(4, -1))
        gen = o[:, C:]
        assert int(gen.min()) >= 0 and int(gen.max()) < 8192
        assert len({tuple(r.tolist()) for r in gen}) > 1


def test_one_caption_and_the_fallbacks_take_the_existing_path(gen_model, tok, monkeypatch):
    from cogview_b200.generation import sampling

    def both(seqs, args, seed=11):
        torch.manual_seed(seed)
        with torch.no_grad():
            got = sampling.filling_sequences(gen_model, seqs, args)
        torch.manual_seed(seed)
        with torch.no_grad():
            want = [sampling.filling_sequence(gen_model, s, args) for s in seqs]
        assert len(got) == len(want) and all(torch.equal(a, b) for a, b in zip(got, want))

    class K(_Args):
        top_k = 200
    both(_captions(tok, [9], 4, 30), K)                          # one caption
    class P(_Args):
        top_k, top_p = 0, 0.9
    both(_captions(tok, [5, 17, 40], 1, 12), P)                   # nucleus sampling
    both(_captions(tok, [5, 17, 40], 24, 12), K)                  # 72 rows
    monkeypatch.setenv("COGVIEW_B200_FAST_DECODE", "0")
    both(_captions(tok, [5, 17, 40], 4, 12), K)


def test_uniform_run_after_a_ragged_run_is_unchanged(gen_model, tok):
    """12 rows: one caption with 12 beams, then three captions of 4, then the first again."""
    from cogview_b200.generation import sampling
    one = _captions(tok, [20], 12, 40, seed=1)[0]
    with torch.no_grad():
        first = sampling.filling_sequence(gen_model, one, _Args)
        runner = gen_model.transformer._kv_pool[12].runner
        launches = runner.graph_launches
        sampling.filling_sequences(gen_model, _captions(tok, [5, 17, 40], 4, 40, seed=2), _Args)
        assert gen_model.transformer._kv_pool[12].runner is runner
        again = sampling.filling_sequence(gen_model, one, _Args)
    assert torch.equal(first, again) and runner.graph_launches == launches and not runner.ragged
