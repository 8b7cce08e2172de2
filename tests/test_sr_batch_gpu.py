"""GPU tests of super-resolving many images in one decode batch: cv_attn_chunk_ragged (a chunk of new tokens per row
against the row's own cached prefix), GPT2Model.chunk_run, filling_sequences on the nine magnify window templates, and
generate.super_resolution_batch end to end.

Tolerances: the kernel against a float64 softmax over each row's own keys, to one bf16 rounding of the output
(2^-8 relative) plus the bf16 rounding of the probabilities that feed the P.V tensor-core product (2^-9 of
sum_k p_k |v_k|) plus 1e-3 absolute; chunk_run's logits against each row run alone through GPT2Model.forward with its
own mems, to 2e-2 of the logit scale (the abs-max LayerNorm scales are taken over the whole batch, so other rows change
them); greedy tokens equal a template's solo run up to the first generated slot whose solo top-2 logit margin is within
that bound (the margin rule of test_caption_batch_gpu.py).
"""
import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu

HD = 64
N_TXT = 101


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


# ----------------------------------------------------------------------------------------------------
# 1. cv_attn_chunk_ragged
# ----------------------------------------------------------------------------------------------------
def _pads(b, cur_len, g):
    """Row 0: no pad; row 1: the whole cache (t_r = 0); the rest random."""
    pads = torch.randint(0, cur_len + 1, (b,), generator=g)
    pads[0] = 0
    if b > 1:
        pads[1] = cur_len
    return pads.to(torch.int32)


@pytest.mark.parametrize("heads", [4, 40])
@pytest.mark.parametrize("b", [1, 5, 16, 64])
@pytest.mark.parametrize("n", [1, 17, 64])
def test_attn_chunk_ragged(ops, n, b, heads):
    h = heads * HD
    for max_len, cur_len in ((1100, 1030), (80, 16)):
        seed = n * 100000 + b * 1000 + heads * 10 + cur_len
        g, gd = torch.Generator().manual_seed(seed), torch.Generator(device="cuda").manual_seed(seed)
        pads = _pads(b, cur_len, g)
        t = (cur_len - pads).tolist()
        cache = torch.randn((b, max_len, 2 * h), generator=gd, device="cuda").to(torch.bfloat16)
        for r in range(b):
            cache[r, t[r]:] = float("nan")                      # never read; only the chunk's slots are written
        qkv = torch.randn((b, n, 3 * h), generator=gd, device="cuda").to(torch.bfloat16)
        before = cache.clone()
        q = qkv[..., :h].double().view(b, n, heads, HD)
        k_new, v_new = qkv[..., h:2 * h], qkv[..., 2 * h:]
        refs, bounds = [], []
        for r in range(b):
            k = torch.cat((before[r, :t[r], :h], k_new[r])).double().view(-1, heads, HD)
            v = torch.cat((before[r, :t[r], h:], v_new[r])).double().view(-1, heads, HD)
            s = torch.einsum("ihd,khd->hik", q[r], k) / HD ** 0.5
            kpos = torch.arange(t[r] + n, device="cuda").view(1, -1)
            qpos = t[r] + torch.arange(n, device="cuda").view(-1, 1)
            s = s.masked_fill((kpos > qpos).unsqueeze(0), float("-inf"))
            pr = torch.softmax(s, dim=-1)
            refs.append(torch.einsum("hik,khd->ihd", pr, v).reshape(n, h))
            # the probabilities enter the P.V tensor-core product rounded to bf16 (relative 2^-9 each), so the
            # context can move by up to 2^-9 * sum_k p_k |v_k|, on top of the output's own bf16 rounding
            bounds.append(2.0 ** -9 * torch.einsum("hik,khd->ihd", pr, v.abs()).reshape(n, h))
        outs = {}
        for nsplit in (None, 1, 7):
            c = before.clone()
            out = ops.attn_chunk_ragged(qkv, c, heads, cur_len, pads.cuda(), nsplit=nsplit)
            torch.cuda.synchronize()
            outs[nsplit] = out
            for r in range(b):
                err = (out[r].double() - refs[r]).abs()
                assert bool((err <= 2.0 ** -8 * refs[r].abs() + bounds[r] + 1e-3).all()), \
                    (max_len, cur_len, nsplit, r, t[r], err.max().item())
                # the chunk lands at t_r .. t_r + n - 1 with the input's bits; every other slot keeps its bits
                want = before[r].clone()
                want[t[r]:t[r] + n, :h], want[t[r]:t[r] + n, h:] = k_new[r], v_new[r]
                assert torch.equal(c[r].view(torch.int16), want.view(torch.int16)), (nsplit, r, t[r])
        if n == 1:       # one query per row: cv_attn_decode's result with row_pad, within tolerance
            c = before.clone()
            dec = ops.attn_decode(qkv.view(b, 3 * h), c, heads, cur_len=cur_len, row_pad=pads.cuda())
            for nsplit, out in outs.items():
                ref = dec.double()
                err = (out.view(b, h).double() - ref).abs()
                bound = torch.cat(bounds).view(b, h)
                assert bool((err <= 2.0 ** -7 * ref.abs() + bound + 2e-3).all()), (nsplit, err.max().item())


def test_attn_chunk_ragged_argument_errors(ops):
    from cogview_b200._lib import CogViewB200Error
    h = 4 * HD
    cache = torch.zeros((2, 64, 2 * h), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(CogViewB200Error, match="1 <= n <= 64"):
        ops.attn_chunk_ragged(torch.zeros((2, 65, 3 * h), dtype=torch.bfloat16, device="cuda"),
                              torch.zeros((2, 200, 2 * h), dtype=torch.bfloat16, device="cuda"), 4, 0)
    with pytest.raises(CogViewB200Error, match="cur_len \\+ n <= max_len"):
        ops.attn_chunk_ragged(torch.zeros((2, 17, 3 * h), dtype=torch.bfloat16, device="cuda"), cache, 4, 48)


# ----------------------------------------------------------------------------------------------------
# 2. GPT2Model.chunk_run
# ----------------------------------------------------------------------------------------------------
CFG = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=256, num_attention_heads=4)


def _model(maxlen, max_seq, seed=31):
    from cogview_b200.model import GPT2Model
    m = GPT2Model(num_layers=CFG["num_layers"], vocab_size=CFG["vocab_size"], hidden_size=CFG["hidden_size"],
                  num_attention_heads=CFG["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=max_seq,
                  max_memory_length=maxlen, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(max_sequence_length=max_seq, seed=seed, **CFG))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    return m


@pytest.fixture(scope="module")
def sr_model():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return _model(1345, 1089)


@pytest.mark.parametrize("lens", [(9, 30, 100), (3, 50, 64, 17, 200, 5)])
def test_chunk_run_matches_each_row_alone(sr_model, lens):
    from cogview_b200.mpu import kv_cache
    model = sr_model
    g = torch.Generator().manual_seed(sum(lens))
    prompts = [torch.randint(0, 8192, (1, n), generator=g).cuda() for n in lens]
    offsets = [n // 2 for n in lens]                          # a different [ROI2] offset per row
    with torch.no_grad():
        mems = []
        for p, o in zip(prompts, offsets):
            pos = torch.arange(p.shape[1], device="cuda").view(1, -1)
            pos = torch.where(pos > o, pos - o, pos)
            _, *m = model(p, pos, torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), device="cuda")), None, None, 0)
            mems.append([x.clone() for x in m])
        bm, row_pad = kv_cache.assemble(model.transformer, mems, [1] * len(lens), 40)
        t = max(lens)
        for step, n in enumerate((17, 5)):
            chunk = torch.randint(0, 8192, (len(lens), n), generator=g).cuda()
            start = [ln + 17 * step for ln in lens]
            pos = torch.stack([torch.arange(s, s + n) - o for s, o in zip(start, offsets)]).cuda()
            logits, bm = model.chunk_run(chunk, pos, bm, row_pad)
            assert logits.shape == (len(lens), CFG["vocab_size"]) and bm[0].shape[1] == t + 17 * step + n
            for r in range(len(lens)):
                lg, *mr = model(chunk[r:r + 1], pos[r:r + 1], 0, None, None, 0, *mems[r])
                mems[r] = [x.clone() for x in mr]
                ls = lg[0, -1]
                scale = ls.abs().max().item()
                err = (logits[r] - ls).abs().max().item()
                print("rows %d, chunk %d, row %d (len %d): logits max|diff| %.3e (scale %.3e)"
                      % (len(lens), n, r, lens[r], err, scale))
                assert err < 2e-2 * scale
                ln = mems[r][0].shape[1]
                for i in range(CFG["num_layers"]):
                    kb, ks = bm[i][r, ln - n:ln].float(), mems[r][i][0, ln - n:ln].float()
                    assert (kb - ks).abs().max().item() < 2e-2 * ks.abs().max().item()
        # a generate run continues every row at its own length after the chunks
        res = model.generate_run(logits[:, :8192].argmax(-1, keepdim=True), pos[:, -1] + 1, bm, 3, 1.0, 1,
                                 [slice(8192, None)], row_pad=row_pad)
        assert res is not None and res[2][0].shape[1] == t + 22 + 3


# ----------------------------------------------------------------------------------------------------
# 3. filling_sequences on the nine magnify windows
# ----------------------------------------------------------------------------------------------------
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


def _texts(tok, lens, g):
    return [torch.tensor([tok['[ROI1]']] + (8192 + torch.randint(0, N_TXT, (n,), generator=g)).tolist()
                         + [tok['[BASE]'], tok['[BOI1]']], device="cuda") for n in lens]


def _window_templates(tok, w, texts, g):
    """The templates magnify builds for window w of each image, with the windows before w already filled (random
    codes standing in for the earlier windows' output)."""
    from cogview_b200.generation.magnify import WINDOWS
    midfix = torch.tensor([tok['[EOI1]'], tok['[ROI2]'], tok['[POS0]'], tok['[BASE]'], tok['[BOI2]']], device="cuda")
    seqs = []
    for text in texts:
        code = torch.randint(0, 8192, (32, 32), generator=g).cuda()
        mag = torch.full((64, 64), -1, dtype=torch.long, device="cuda")
        for i, j, line in WINDOWS[:w]:
            mag[16 * i:16 * i + line, 16 * j:16 * (j + 2)] = torch.randint(0, 8192, (line, 32), generator=g).cuda()
        i, j, line = WINDOWS[w]
        ctx = torch.cat([text, code[8 * i:8 * (i + 2), 8 * j:8 * (j + 2)].reshape(-1), midfix])
        seqs.append(torch.cat([ctx, mag[16 * i:16 * i + line, 16 * j:16 * (j + 2)].reshape(-1)]))
    return seqs


def _decisive_prefix(model, row, C, offset, gen_mask):
    """Length of the leading part of `row` that a greedy run must reproduce: up to the first generated slot (after the
    context's own first draw) whose top-2 image-code margin in a teacher-forced forward is within 2e-2 of the logit
    scale."""
    s = row.shape[0]
    pos = torch.arange(s - 1, device="cuda")
    pos = torch.where(pos > offset, pos - offset, pos).view(1, -1)
    with torch.no_grad():
        lg, *_ = model(row[:-1].view(1, -1), pos, torch.tril(torch.ones((1, 1, s - 1, s - 1), device="cuda")), None,
                       None, 0)
    lg = lg[0, C:, :8192].float()                               # predicts slots C + 1 ..
    top = lg.topk(2, dim=-1).values
    bad = ((top[:, 0] - top[:, 1] <= 2e-2 * lg.abs().amax(-1)) & gen_mask[C + 1:]).nonzero()
    return C + 1 + (int(bad[0]) if bad.numel() else s - C - 1)


@pytest.mark.parametrize("w", range(9))
def test_greedy_rows_follow_each_window_template_alone(sr_model, tok, w):
    from cogview_b200.generation import sampling
    n_img = 3 + (13 * w) // 8                                   # 3 .. 16 images
    g = torch.Generator().manual_seed(100 + w)
    texts = _texts(tok, [2 + (7 * r) % 40 for r in range(n_img)], g)
    seqs = _window_templates(tok, w, texts, g)
    with torch.no_grad():
        out = sampling.filling_sequences(sr_model, seqs, _Args)
        solo = [sampling.filling_sequence(sr_model, s, _Args) for s in seqs]
    compared = 0
    for o, s, seq in zip(out, solo, seqs):
        assert o.shape == s.shape == (1, len(seq))
        C, offset, _ = sampling._scan_context(seq.tolist(), tok)
        gen = seq < 0
        k = _decisive_prefix(sr_model, s[0], C, offset, gen)
        assert torch.equal(o[0, :k], s[0, :k]), (w, C, k)
        assert torch.equal(o[0, ~gen], seq[~gen])
        compared += int(gen[:k].sum())
    print("window %d, %d images: %d generated tokens compared" % (w, n_img, compared))
    assert compared > 0


# ----------------------------------------------------------------------------------------------------
# 4. generate.super_resolution_batch
# ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def vq():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import vqvae
    model = vqvae.new_model()
    model.load_state_dict(recipes.vqvae_state_dict(seed=0))
    return model.cuda().eval()


def _sr_seqs(tok, lens, g, same=False):
    from cogview_b200 import generate
    out = []
    for n in lens:
        if not out or not same:
            text = (8192 + torch.randint(0, N_TXT, (n,), generator=g)).tolist()
            src = torch.randint(0, 8192, (1024,), generator=g).tolist()
        out.append(torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['super-resolution'], [text, src],
                                                     tokenizer=tok), dtype=torch.long, device="cuda"))
    return out


def test_super_resolution_batch_identical_rows(sr_model, vq, tok):
    from cogview_b200 import generate, vqvae
    seqs = _sr_seqs(tok, [6, 6, 6], torch.Generator().manual_seed(41), same=True)
    codes, imgs = generate.super_resolution_batch(sr_model, vq, _Args, seqs)
    assert codes.shape == (3, 4096) and imgs.shape == (3, 3, 512, 512)
    assert int(codes.min()) >= 0 and int(codes.max()) < 8192
    assert torch.equal(codes[1], codes[0]) and torch.equal(codes[2], codes[0])
    with torch.no_grad():
        assert torch.equal(imgs, torch.cat([vqvae.code2img(vq, c.view(1, 64, 64)) for c in codes]))


def test_super_resolution_batch_is_super_resolution_without_a_batch(sr_model, vq, tok, monkeypatch):
    """One image, and the per-template fallback (COGVIEW_B200_FAST_DECODE=0): bit-equal to super_resolution."""
    from cogview_b200 import generate
    g = torch.Generator().manual_seed(43)
    one = _sr_seqs(tok, [9], g)
    codes, imgs = generate.super_resolution_batch(sr_model, vq, _Args, one)
    want_c, want_i = generate.super_resolution(sr_model, vq, _Args, one[0])
    assert torch.equal(codes, want_c) and torch.equal(imgs, want_i)

    monkeypatch.setenv("COGVIEW_B200_FAST_DECODE", "0")
    two = _sr_seqs(tok, [4, 15], g)
    codes, imgs = generate.super_resolution_batch(sr_model, vq, _Args, two)
    for r, seq in enumerate(two):
        want_c, want_i = generate.super_resolution(sr_model, vq, _Args, seq)
        assert torch.equal(codes[r:r + 1], want_c) and torch.equal(imgs[r:r + 1], want_i)
