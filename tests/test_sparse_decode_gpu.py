"""GPU tests of sparse inference on the device (is_sparse == 2 inside generate_run): the per-step key index plan
(cv_sparse_plan), the gathered decode attention (cv_attn_decode_gather) and the generation loop built on them.

Reference semantics: mpu/sparse_transformer.py:498-520 (index bookkeeping: trailing window of query_window *
key_window_times keys, all text positions before it, num_pivot_now = max_text + int((left_boundary - max_text) * num_pivot /
max_sequence_length) entries), :591-600 (fresh random image pivots per layer per token) and :727-750 (softmax over the
gathered keys).  The device draws the random subset with counter-based keys instead of Python's random.sample: the tests pin
everything that does not depend on the stream (membership, counts, distinctness, freshness) and the attention itself."""
import math

import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu


def test_sparse_plan_structure_and_freshness():
    from cogview_b200 import ops
    L, b, maxlen, window, num_pivot, max_seq = 6, 3, 1200, 96, 300, 1200
    g = torch.Generator().manual_seed(0)
    is_txt = torch.zeros((b, maxlen + 1), dtype=torch.uint8)
    n_txt = [17, 30, 24]
    for i in range(b):
        is_txt[i, torch.randperm(400, generator=g)[:n_txt[i]]] = 1
    is_txt = is_txt.cuda()
    idx = torch.full((L, b, num_pivot + window), -1, dtype=torch.int32, device="cuda")
    n_dev = torch.zeros(1, dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    seed = torch.tensor([12345], dtype=torch.int64, device="cuda")
    for t in (10, 95, 96, 500, 1100):
        cur = torch.tensor([t], dtype=torch.int32, device="cuda")
        ops.sparse_plan(is_txt, cur, L, window, num_pivot, max_seq, seed, idx, n_dev, err)
        torch.cuda.synchronize()
        assert err.item() == 0
        key_length = t + 1
        lb = max(0, key_length - window)
        counts = [int(is_txt[i, :lb].sum()) for i in range(b)]
        max_text = max(counts) if lb > 0 else 0
        want_piv = max_text + int((lb - max_text) * (num_pivot / max_seq))         # :508-510
        n = n_dev.item()
        assert n == want_piv + key_length - lb
        got = idx.cpu()
        for l in range(L):
            for i in range(b):
                row = got[l, i, :n].tolist()
                piv, win = row[:want_piv], row[want_piv:]
                assert win == list(range(lb, key_length))                           # trailing window, the new token last
                assert len(set(piv)) == want_piv and all(0 <= p < lb for p in piv)  # distinct positions before the window
                txt = set(torch.nonzero(is_txt[i, :lb].cpu()).view(-1).tolist())
                assert txt <= set(piv)                                              # every text position is a pivot
                assert len(set(piv) - txt) == want_piv - counts[i]                  # the rest are image positions
        if want_piv > max_text + 8:
            a, c = set(got[0, 0, :want_piv].tolist()), set(got[1, 0, :want_piv].tolist())
            assert a != c                                                           # fresh per layer
            ops.sparse_plan(is_txt, cur, L, window, num_pivot, max_seq, seed + 1, idx, n_dev, err)
            torch.cuda.synchronize()
            assert set(idx[0, 0, :want_piv].cpu().tolist()) != a                    # and per seed / run
    # uniformity of the image sample: every image position before the window is chosen about equally often
    t = 1100
    cur = torch.tensor([t], dtype=torch.int32, device="cuda")
    lb = t + 1 - window
    hits = torch.zeros(lb)
    reps = 60
    for r in range(reps):
        ops.sparse_plan(is_txt, cur, L, window, num_pivot, max_seq, seed + 100 + r, idx, n_dev, err)
        n = n_dev.item()
        piv = idx[:, 0, :n - window].cpu().long().view(-1)
        hits += torch.bincount(piv, minlength=lb).float()
    img = ~is_txt[0, :lb].cpu().bool()
    k_img = (n - window) - int(is_txt[0, :lb].sum())
    p = k_img / int(img.sum())
    draws = reps * L
    freq = hits[img] / draws
    assert abs(freq.mean().item() - p) < 1e-6
    assert (freq - p).abs().max().item() < 6 * math.sqrt(p * (1 - p) / draws)      # no position favoured


def _fill(is_sparse, num_pivot, monkeypatch, pivots="device", text_gen=False):
    """Greedy filling of 60 tokens after a short context with a 4 x 4 = 16-key window: image tokens after [BOI1], or text
    tokens (no [BOI1] in the context: generation/sampling.py starts in the text vocabulary) when text_gen."""
    from cogview_b200.generation import sampling
    from cogview_b200.model import GPT2Model
    monkeypatch.setenv("COGVIEW_B200_SPARSE_PIVOTS", pivots)
    cfg = recipes.CONFIG1
    m = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                  num_attention_heads=cfg["num_attention_heads"], embedding_dropout_prob=0.0, attention_dropout_prob=0.0,
                  output_dropout_prob=0.0, max_sequence_length=cfg["max_sequence_length"],
                  max_memory_length=cfg["max_sequence_length"], checkpoint_activations=False, query_window=4,
                  key_window_times=4, num_pivot=num_pivot)
    m.load_state_dict(recipes.gpt2_state_dict(**cfg))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"

    class A:
        temperature, top_p, top_k = 1.0, 0.0, 1          # greedy: no randomness in the draw
        img_tokenizer_num_tokens = recipes.IMG_VOCAB
    A.is_sparse = is_sparse
    tok = sampling.get_tokenizer(A)
    g = torch.Generator().manual_seed(3)
    text = torch.randint(recipes.IMG_VOCAB, recipes.IMG_VOCAB + 100, (10,), generator=g).tolist()
    seq = [tok['[ROI1]']] + text + ([] if text_gen else [tok['[BASE]'], tok['[BOI1]']]) + [-2] * 60
    with torch.no_grad():
        out = sampling.filling_sequence(m, torch.tensor(seq, dtype=torch.long, device="cuda"), A)
    return out.cpu(), m


def test_sparse_generation_on_the_device(monkeypatch):
    """(1) When the pivot budget covers every earlier position (num_pivot = max_sequence_length), pivots + window is every
    key, so the device-side sparse run must reproduce the dense greedy tokens — pins the text flags, the plan, the window,
    the append and the hand-over of tokens between steps.  (2) With a small budget the run completes on the graph path (one
    plan launch + gather attention per layer per token) and stays inside the image vocabulary."""
    dense, _ = _fill(0, 128, monkeypatch)
    sparse_all, m = _fill(2, recipes.CONFIG1["max_sequence_length"], monkeypatch)
    assert dense.shape == sparse_all.shape
    agree = (dense == sparse_all).float().mean().item()
    print("sparse (all positions as pivots) vs dense greedy tokens: %.3f equal" % agree)
    assert agree > 0.97                                  # bf16 ties aside
    runner = m.transformer._kv.runner
    assert runner.replays >= 59 and runner.is_txt is not None
    few, m2 = _fill(2, 24, monkeypatch)
    r2 = m2.transformer._kv.runner
    assert r2.replays >= 59 and int(r2.plan_err.item()) == 0
    gen = few[:, -60:]
    assert int(gen.max()) < recipes.IMG_VOCAB and few.shape == dense.shape
    n = int(r2.n_keys.item())
    assert n < few.shape[1]                              # a strict subset of the keys was attended at the last step


def test_sparse_generation_tracks_text_flags_of_generated_tokens(monkeypatch):
    """Generated TEXT tokens must be flagged as text for the following steps (all text positions are pivots,
    mpu/sparse_transformer.py:504-510): with every earlier position a text position the key list is every key, so the run
    must reproduce the dense greedy tokens although only half of the IMAGE positions would be kept (num_pivot /
    max_sequence_length = 0.5) — a flag written at the wrong position, or not at all, changes the attended set."""
    dense, _ = _fill(0, 64, monkeypatch, text_gen=True)
    sparse, m = _fill(2, 64, monkeypatch, text_gen=True)
    gen = sparse[:, -60:]
    assert int(gen.min()) >= recipes.IMG_VOCAB            # text tokens were generated
    agree = (dense == sparse).float().mean().item()
    print("sparse text generation vs dense greedy tokens: %.3f equal" % agree)
    assert agree > 0.97
    r = m.transformer._kv.runner
    T = sparse.shape[1]
    flags = r.is_txt[:, :T - 1].cpu().bool()               # the last sampled token is flagged when it is fed
    assert torch.equal(flags, sparse[:, :T - 1] >= recipes.IMG_VOCAB)
    assert int(r.plan_err.item()) == 0
