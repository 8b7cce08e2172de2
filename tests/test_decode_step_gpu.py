"""GPU tests of the graph-replayed decode step (DecodeRunner, mpu/decode.py) and the fused sampling epilogue
(cv_sample_topk, csrc/sample.cu).

* the step replayed from a CUDA graph against its eager launch, and a weight change after the first generation
  picked up by the next sequence (the step's numerics against a second route are tested in
  test_decode_mid_gpu.py::test_graph_step_matches_the_general_route, for 1..64 sequences);
* the sampling kernel against the reference semantics (generation/sampling.py:24-33,157-183) restated with torch:
  same kept set (ties at the k-th value included), same probabilities, draws distributed accordingly.
"""
import math

import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu


def _model(cfg, maxlen):
    from cogview_b200.model import GPT2Model
    m = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                  num_attention_heads=cfg["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=maxlen,
                  max_memory_length=maxlen, checkpoint_activations=False)
    sd = recipes.gpt2_state_dict(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"],
                                 hidden_size=cfg["hidden_size"], max_sequence_length=maxlen, seed=7)
    m.load_state_dict(sd)
    return m.cuda().bfloat16().eval()


CFG_TINY = dict(num_layers=2, vocab_size=58240, hidden_size=256, num_attention_heads=4)


def test_decode_step_graph_replay_and_weight_refresh():
    """The step under CUDA-graph capture (the production mode) reproduces the eager launch, and a weight change
    after the first generation is picked up (parameters gathered again, captured graph rebuilt)."""
    from cogview_b200.mpu import kv_cache
    from cogview_b200.mpu.decode import DecodeRunner
    model = _model(CFG_TINY, 128)
    tr = model.transformer
    b, t = 4, 9
    base = None
    outs = []
    for use_graph in (False, True):
        c = kv_cache._Caches(tr, b, torch.device("cuda"))
        if base is None:
            base = torch.randn(c.buf.shape, device="cuda").to(torch.bfloat16)
        c.buf.copy_(base)
        c.t = t
        r = DecodeRunner(model, c, use_graph=use_graph)
        ids = torch.arange(b, device="cuda").view(b, 1) + 5
        pos = torch.full((b, 1), t, dtype=torch.long, device="cuda")
        with torch.no_grad():
            a = r.step(ids, pos, t).clone()
            bb = r.step(ids + 1, pos + 1, t + 1).clone()
        outs.append((a, bb, r, c))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    # change a weight in place: the next sequence must see it
    a, _, r, c = outs[1]
    with torch.no_grad():
        model.transformer.final_layernorm.weight.mul_(2.0)
        ids = torch.arange(b, device="cuda").view(b, 1) + 5
        pos = torch.full((b, 1), t, dtype=torch.long, device="cuda")
        c.buf.copy_(base)
        a2 = r.step(ids, pos, t).clone()          # t <= last_t: parameters are re-checked
    assert not torch.allclose(a, a2)


def _ref_probs(logits, temperature, top_k, valid):
    lg = logits.clone() / temperature
    mask = torch.ones_like(lg, dtype=torch.bool)
    for lo, hi in valid:
        mask[:, lo:hi] = False
    lg[mask] = -float("inf")
    if top_k > 0:
        kth = torch.topk(lg, top_k)[0][..., -1, None]
        lg[lg < kth] = -float("inf")
    return torch.softmax(lg, dim=-1)


@pytest.mark.parametrize("valid,top_k,temperature", [([(0, 8192)], 200, 1.0), ([(8192, 58192)], 200, 0.8),
                                                     ([(0, 8192), (58192, 58240)], 50, 1.3), ([(0, 58240)], 0, 1.0),
                                                     ([(0, 8192)], 1, 1.0), ([(0, 8192)], 9000, 1.0)])
def test_sample_topk_distribution_matches_reference_semantics(valid, top_k, temperature):
    from cogview_b200 import ops
    torch.manual_seed(0)
    b, V = 4, 58240
    logits = (torch.randn((b, V), device="cuda") * 3.0).contiguous()
    # ties exactly at the top-k threshold: `logits < kth` keeps all of them
    lo0 = valid[0][0]
    srt = torch.sort(logits[0, valid[0][0]:valid[0][1]], descending=True)[0]
    if 1 < top_k < 500:
        logits[0, lo0 + 3] = srt[top_k - 1]
        logits[0, lo0 + 11] = srt[top_k - 1]
    keep = logits.clone()
    ref = _ref_probs(logits, temperature, top_k, valid)
    nxt, probs = ops.sample_topk(logits, temperature, top_k, valid, seed=123, want_probs=True)
    torch.cuda.synchronize()
    assert torch.equal(logits, keep), "the kernel must not modify the logits"
    assert torch.equal(probs > 0, ref > 0), "kept set differs from top_k_logits"
    assert (probs - ref).abs().max().item() < 1e-6 + 1e-4 * ref.max().item()
    assert bool(((nxt >= 0) & (nxt < V)).all()) and bool((ref.gather(1, nxt.view(-1, 1)) > 0).all())
    # draws follow the distribution: 4000 draws per row through the device-side step counter
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
        ops.sample_topk(logits, temperature, top_k, valid, seed_dev=seed_dev, step=step, next_ids=ids, out_tokens=out,
                        score_acc=score, pos=pos, cur_len=cur, done=done)
    torch.cuda.synchronize()
    assert int(step) == n and int(cur) == n and bool((pos == n).all()) and int(done) == 0
    assert torch.equal(out[:, -1], ids)
    lp = torch.log(ref.gather(1, out)).sum(1)
    assert torch.allclose(score, lp, rtol=1e-3, atol=1e-2)
    for r in range(b):
        p = ref[r]
        top = torch.topk(p, 5)
        cnt = torch.bincount(out[r], minlength=V).float()
        assert float(cnt[p == 0].sum()) == 0
        for pv, iv in zip(top.values.tolist(), top.indices.tolist()):
            sd = math.sqrt(n * pv * (1 - pv)) + 1.0
            assert abs(float(cnt[iv]) - n * pv) < 5 * sd, (r, iv, pv, float(cnt[iv]))
