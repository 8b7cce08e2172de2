"""Host logic of batched post-selection: inverse_prompt_scores' grouping, [PAD] padding, scored positions, order
restoration and layout check, and rerank's choice of the best candidates — with stand-in models, no GPU."""
import pytest
import torch

from cogview_b200 import generate as gen
from cogview_b200.generation import sampling

N_IMG, N_TXT = 8192, 300


class Args:
    is_sparse = 0
    img_tokenizer_num_tokens = N_IMG
    max_inference_batch_size = 4


@pytest.fixture
def tok(monkeypatch):
    t = sampling.TokenLayout(img_tokens=N_IMG, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


class StandIn:
    """token_logprobs of a position-wise model (embedding table + position term, tied output): no attention, so a
    row's scores cannot depend on the padding or on the other rows of its group."""

    def __init__(self, vocab, seed=3):
        self.table = 0.15 * torch.randn(vocab, 16, generator=torch.Generator().manual_seed(seed))
        self.calls = []

    def eval(self):
        return self

    def token_logprobs(self, input_ids, position_ids, attention_mask, score_index, targets, vocab_begin=0,
                       vocab_end=None):
        assert not torch.is_grad_enabled()
        self.calls.append(dict(tokens=input_ids.clone(), index=score_index.clone(), targets=targets.clone(),
                               window=(vocab_begin, vocab_end)))
        b, s = input_ids.shape
        assert position_ids.shape[-1] == s and attention_mask.shape[-1] == s
        h = self.table[input_ids] + 0.01 * position_ids.unsqueeze(-1).float()
        lg = h.view(b * s, -1)[score_index] @ self.table.t()
        lg[:, :vocab_begin] = -float("inf")
        return torch.log_softmax(lg, -1).gather(1, targets.view(-1, 1)).view(-1)


def _formula(table, row):
    """inverse_prompt_score's sum written out for one row"""
    botext = 2 + 1024 + 1
    total = 0.0
    for t in range(botext, len(row) - 1):
        lg = (table[row[t]] + 0.01 * t) @ table.t()
        lg[:N_IMG] = -float("inf")
        total += torch.log_softmax(lg, -1)[row[t + 1]].item()
    return total


def _rows(tok, n, text_lens, seed=5):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        text = (N_IMG + torch.randint(0, N_TXT, (text_lens[i % len(text_lens)],), generator=g)).tolist()
        codes = torch.randint(0, N_IMG, (1024,), generator=g).tolist()
        out.append(torch.tensor(gen.build_query(gen.QUERY_TEMPLATES['post-selection'], [codes, text], tok)))
    return out


def test_groups_pad_and_restore_order(tok):
    rows = _rows(tok, 10, [3, 7, 1, 12])
    model = StandIn(tok.num_tokens)
    scores = sampling.inverse_prompt_scores(model, rows, Args)
    assert scores.shape == (10,) and scores.dtype == torch.float32
    assert [c["tokens"].shape[0] for c in model.calls] == [4, 4, 2]
    for c in model.calls:
        assert c["window"] == (N_IMG, None)
    # padding at the end with [PAD], rows in input order, only caption positions scored
    first = model.calls[0]
    L = first["tokens"].shape[1]
    assert L == max(len(r) for r in rows[:4])
    for i, r in enumerate(rows[:4]):
        assert torch.equal(first["tokens"][i, :len(r)], r)
        assert bool((first["tokens"][i, len(r):] == tok['[PAD]']).all())
    want_index = [i * L + t for i, r in enumerate(rows[:4]) for t in range(1027, len(r) - 1)]
    assert first["index"].tolist() == want_index
    assert first["targets"].tolist() == [first["tokens"].view(-1)[j + 1].item() for j in want_index]
    for i, r in enumerate(rows):
        want = _formula(model.table, r.tolist())
        assert abs(scores[i].item() - want) < 1e-4 * abs(want) + 1e-5, (i, scores[i].item(), want)


def test_a_2d_tensor_and_group_sizes_agree(tok):
    rows = _rows(tok, 6, [5])
    model = StandIn(tok.num_tokens)
    a = sampling.inverse_prompt_scores(model, torch.stack(rows), Args)
    Args1 = type("Args1", (Args,), {"max_inference_batch_size": 64})
    b = sampling.inverse_prompt_scores(model, rows, Args1)
    assert [c["tokens"].shape[0] for c in model.calls] == [4, 2, 6]
    assert torch.allclose(a, b, rtol=1e-6, atol=1e-6)
    # the batched scorer plugs into post_selection in place of inverse_prompt_score
    c = gen.post_selection(model, Args, torch.stack(rows[:4]), score=sampling.inverse_prompt_scores)
    assert torch.allclose(c, a[:4], rtol=1e-6, atol=1e-6)


def test_layout_is_checked(tok):
    rows = _rows(tok, 3, [4])
    bad = rows[1].clone()
    bad[1027] = tok['[SEP]']
    with pytest.raises(AssertionError):
        sampling.inverse_prompt_scores(StandIn(tok.num_tokens), [rows[0], bad, rows[2]], Args)
    with pytest.raises(AssertionError):     # no caption token to score
        sampling.inverse_prompt_scores(StandIn(tok.num_tokens), [rows[0][:1028]], Args)
    SparseArgs = type("SparseArgs", (Args,), {"is_sparse": 2})
    with pytest.raises(NotImplementedError):
        sampling.inverse_prompt_scores(StandIn(tok.num_tokens), rows, SparseArgs)


def test_rerank_keeps_the_best_with_ties_to_the_lower_index(tok, monkeypatch):
    g = torch.Generator().manual_seed(9)
    texts = [(N_IMG + torch.randint(0, N_TXT, (n,), generator=g)).tolist() for n in (4, 9)]
    seqs = [torch.tensor(gen.build_query(gen.QUERY_TEMPLATES['text2image'], [t], tok)) for t in texts]
    num, keep = 5, 3
    drawn = []
    for seq in seqs:
        rows = seq.unsqueeze(0).repeat(num, 1)
        rows[:, -1024:] = torch.randint(0, N_IMG, (num, 1024), generator=g)
        drawn.append((rows, torch.arange(num, dtype=torch.float32).view(num, 1, 1, 1).expand(num, 3, 2, 2) + 10 * len(drawn)))
    monkeypatch.setattr(gen, "generate_images_batch", lambda m, vq, a, s, num: drawn)
    fixed = torch.tensor([1.0, 3.0, 3.0, -2.0, 3.0, 0.5, 0.5, 2.0, 0.5, -1.0])
    seen = []

    def fake_scores(model, queries, args):
        seen.append([q.clone() for q in queries])
        return fixed.clone()
    monkeypatch.setattr(gen, "inverse_prompt_scores", fake_scores)
    out = gen.rerank(object(), StandIn(tok.num_tokens), None, Args, seqs, num=num, keep=keep)
    assert len(out) == 2
    # the queries are every caption's post-selection rows, in caption order, with that caption's text
    assert len(seen[0]) == 2 * num
    for c, (rows, _) in enumerate(drawn):
        want = gen.post_selection_rows(rows, texts[c], tok)
        assert torch.equal(torch.stack(seen[0][c * num:(c + 1) * num]), want)
    assert out[0].index.tolist() == [1, 2, 4] and out[1].index.tolist() == [2, 0, 1]
    for c, r in enumerate(out):
        assert torch.equal(r.all_scores, fixed[c * num:(c + 1) * num])
        assert torch.equal(r.scores, r.all_scores[r.index])
        assert torch.equal(r.rows, drawn[c][0][r.index]) and torch.equal(r.images, drawn[c][1][r.index])
