"""Host logic of "draw many, keep the best" (generate_samples.py:246-270) and of the K|V-cache pool that serves it:
post-selection queries built from generated rows, scores chunked by max_inference_batch_size and checked against
the formula written out, and the byte budget of the per-batch-size cache pool."""
import pytest
import torch


def test_post_selection_rows_and_chunked_scores():
    from cogview_b200 import generate as gen
    from cogview_b200.generation import sampling

    class Args:
        is_sparse = 0
        img_tokenizer_num_tokens = 8192
        max_inference_batch_size = 4

    tok = sampling.get_tokenizer(Args)
    vocab = tok.num_tokens
    g = torch.Generator().manual_seed(11)
    text = torch.randint(8192, 58192, (7,), generator=g).tolist()
    template = gen.build_query(gen.QUERY_TEMPLATES['text2image'], [text], tok)
    rows = torch.tensor(template).unsqueeze(0).repeat(8, 1)
    codes = torch.randint(0, 8192, (8, 1024), generator=g)
    rows[:, -1024:] = codes                                          # what generate_images_once returns
    seq = gen.post_selection_rows(rows, text, tok)
    assert seq.shape == (8, 2 + 1024 + 2 + 7) and seq.dtype == torch.long
    for b in range(8):
        assert seq[b].tolist() == ([tok['[BASE]'], tok['[BOI1]']] + codes[b].tolist() + [tok['[EOI1]'], tok['[ROI1]']]
                                   + text)

    table = 0.15 * torch.randn(vocab, 32, generator=g)
    batches = []

    class StandIn(torch.nn.Module):
        def forward(self, tokens, position_ids, attention_mask, txt, img, is_sparse, *mems):
            batches.append(tokens.shape[0])
            h = table[tokens] + 0.01 * position_ids.unsqueeze(-1).float()
            return (h @ table.t(),)

    scores = gen.post_selection(StandIn(), Args, seq)
    assert scores.shape == (8,) and batches == [4, 4]
    botext = 2 + 1024 + 1
    for b in (0, 3, 4, 7):
        total = 0.0
        for t in range(botext, seq.shape[1] - 1):
            lg = (table[seq[b, t]] + 0.01 * t) @ table.t()
            lg[:8192] = -float('inf')
            total += torch.log_softmax(lg, -1)[seq[b, t + 1]].item()
        assert abs(scores[b].item() - total) < 1e-3 * abs(total), (b, scores[b].item(), total)
    # fewer rows than one group: a single call; a ragged count is refused as in generate_images_once
    del batches[:]
    assert gen.post_selection(StandIn(), Args, seq[:3]).shape == (3,) and batches == [3]
    with pytest.raises(AssertionError):
        gen.post_selection(StandIn(), Args, seq[:6])
    # keeping the best k
    best = scores.topk(2).indices.tolist()
    assert scores[best[0]] == scores.max() and len(set(best)) == 2


class _Owner:
    """what kv_cache.prepare reads of GPT2ParallelTransformer"""

    def __init__(self, hidden, layers, maxlen):
        self.hidden_size = hidden
        self.layers = [None] * layers
        self.max_memory_length = maxlen
        self.position_embeddings = torch.nn.Embedding(4, hidden)


def test_kv_pool_keeps_batch_sizes_within_its_byte_budget(monkeypatch):
    from cogview_b200.mpu import kv_cache
    owner = _Owner(hidden=8, layers=2, maxlen=16)
    per_seq = kv_cache.cache_bytes(owner, 1)
    assert per_seq == 2 * 16 * 16 * 2 and kv_cache.cache_bytes(owner, 64) == 64 * per_seq
    monkeypatch.setattr(kv_cache, "POOL_BYTE_BUDGET", 40 * per_seq)
    c1 = kv_cache.prepare(owner, [], 1, 4)
    c4 = kv_cache.prepare(owner, [], 4, 1)
    assert set(owner._kv_pool) == {1, 4}                            # small caches live side by side
    assert kv_cache.prepare(owner, [], 1, 4) is c1                  # and are reused
    c32 = kv_cache.prepare(owner, [], 32, 1)
    assert set(owner._kv_pool) == {1, 4, 32}                        # 37 sequences: still within the budget
    # 64 more would not fit: the largest other caches go first, until the rest fits
    c64 = kv_cache.prepare(owner, [], 64, 1)
    assert set(owner._kv_pool) == {64} and owner._kv is c64
    # the budget never refuses the cache that is asked for, and beams expanded from a dropped cache are copied
    c4.buf.copy_(torch.arange(c4.buf.numel()).view(c4.buf.shape) % 251)
    views = c4.views()
    c32b = kv_cache.prepare(owner, [m.repeat(8, 1, 1) for m in views], 32, 1)
    assert c32b is not c32 and set(owner._kv_pool) == {32} and c32b.t == views[0].size(1)
    assert torch.equal(c32b.buf[0, :4, :c32b.t], c4.buf[0, :, :c32b.t])
