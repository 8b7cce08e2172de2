"""GPU parity of sparse TRAINING attention (SURVEY §8 row a7: sparse_attention + _chunk,
mpu/sparse_transformer.py:675-725, :629-650, pivot mask :491-496 / :569) — cv_attn_sparse_fwd / cv_attn_sparse_bwd.

* forward against tests/golden/attention.npz:sparse_train, the UNMODIFIED reference's output (s = 512, w = 64,
  times = 3, 96 pivots, 2 x 3 heads), and against the oracle restatement on bf16-rounded inputs;
* a 2-layer GPT2Model training step with is_sparse = 1 (fresh pivots per checkpointed layer in the reference's
  random.sample order) against the oracle evaluated with the same pivots.
Tolerances (bf16 tensor-core math vs the fp32 oracle): 2e-2 of the output scale forward, 4e-2 of each gradient's scale.
The kernels themselves are bounded element by element in tests/test_attention_sparse_gpu.py."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import cogview_oracle as O
from oracle import recipes

pytestmark = pytest.mark.gpu


def _rmask(s, w, times):
    g = s // w
    tmp = torch.ones((g - times + 1, w, w))
    tmp = torch.tril(1 - torch.block_diag(*tmp))
    return torch.nn.functional.pad(tmp, (0, (times - 1) * w, (times - 1) * w, 0))


def test_sparse_forward_matches_reference_golden(golden_dir):
    from cogview_b200.mpu.sparse_transformer import sparse_attention
    g = np.load(os.path.join(golden_dir, "attention.npz"))
    b, nh, s, hn, w, times, n_piv, _ = [int(x) for x in g["dims"]]
    gen = torch.Generator().manual_seed(int(g["seed"]))
    q, k, v = (torch.randn((b, nh, s, hn), generator=gen) for _ in range(3))
    pivot_idx = torch.from_numpy(g["pivot_idx"])
    out = sparse_attention(q.cuda().bfloat16(), k.cuda().bfloat16(), v.cuda().bfloat16(), pivot_idx.cuda(), None, w,
                           times).float().cpu()
    ref = g["sparse_train"]
    scale = np.abs(ref).max()
    err = np.abs(out.numpy()[:, :, ::7] - ref).max()
    print("sparse fwd vs reference golden: max|diff| %.3e (scale %.3e)" % (err, scale))
    assert err < 2e-2 * scale
    # and against the oracle on the same bf16-rounded inputs (removes the input rounding from the comparison)
    qb, kb, vb = (t.bfloat16().float() for t in (q, k, v))
    pam = _rmask(s, w, times).expand(b, s, s).gather(dim=-1, index=pivot_idx.unsqueeze(1).expand(b, s, n_piv))
    o = O.sparse_attention(qb, kb, vb, pivot_idx, pam, w, times)
    assert (out - o).abs().max().item() < 1e-2 * o.abs().max().item()


def test_model_sparse_training_step_matches_oracle():
    """GPT2Model(..., checkpoint_activations=True) forward + loss + backward with is_sparse = 1 against the oracle run
    with the SAME pivots (Python `random` is re-seeded before each side: the model draws fresh pivots per layer in
    the reference's order, mpu/sparse_transformer.py:556-565)."""
    from cogview_b200 import mpu
    from cogview_b200.model import GPT2Model
    cfg = dict(num_layers=2, vocab_size=58240, hidden_size=256, num_attention_heads=4, max_sequence_length=256)
    s, w, times, n_piv = 256, 64, 2, 48
    sd32 = recipes.gpt2_state_dict(seed=21, **cfg)
    m = GPT2Model(num_layers=2, vocab_size=cfg["vocab_size"], hidden_size=256, num_attention_heads=4,
                  embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                  max_sequence_length=s, max_memory_length=0, checkpoint_activations=True, checkpoint_num_layers=1,
                  query_window=w, key_window_times=times, num_pivot=n_piv)
    m.load_state_dict(sd32)
    m = m.cuda().bfloat16().train()
    tokens = recipes.text_image_tokens(2, 32, s - 32, seed=3)
    labels = torch.roll(tokens, -1, dims=1)
    pos = torch.arange(s).unsqueeze(0).expand(2, -1).contiguous()
    img = tokens < recipes.IMG_VOCAB
    random.seed(77)
    logits, *_ = m(tokens.cuda(), pos.cuda(), torch.tril(torch.ones((1, 1, s, s), device="cuda")), (~img).cuda(),
                   img.cuda(), 1)
    loss = mpu.vocab_parallel_cross_entropy(logits.contiguous().float(), labels.cuda()).mean()
    loss.backward()
    # oracle with the same per-layer pivots
    random.seed(77)
    img_all = [img[i].nonzero(as_tuple=False).view(-1) for i in range(2)]
    txt_all = [(~img)[i].nonzero(as_tuple=False).view(-1) for i in range(2)]
    from cogview_b200.mpu.sparse_transformer import GPT2ParallelTransformer
    pivots = [GPT2ParallelTransformer.sample_pivot_idx(img_all, txt_all, n_piv) for _ in range(2)]
    sdr = {k: v.to(torch.bfloat16).float().requires_grad_(True) for k, v in sd32.items()}
    rm = _rmask(s, w, times)
    x = torch.nn.functional.embedding(tokens, sdr["word_embeddings.weight"]) + \
        torch.nn.functional.embedding(pos, sdr["transformer.position_embeddings.weight"])
    for li in range(2):
        pam = rm.expand(2, s, s).gather(dim=-1, index=pivots[li].unsqueeze(1).expand(2, s, n_piv))
        x = O.transformer_layer(sdr, li, x, pam, 4, is_sparse=1, pivot_idx=pivots[li], query_window=w,
                                key_window_times=times)
    xf = O.layernorm_absmax(x, sdr["transformer.final_layernorm.weight"], sdr["transformer.final_layernorm.bias"])
    o_logits = torch.nn.functional.linear(xf, sdr["word_embeddings.weight"])
    o_loss = O.vocab_parallel_cross_entropy(o_logits, labels).mean()
    o_loss.backward()
    scale = o_logits.abs().max().item()
    err = (logits.float().cpu() - o_logits.detach()).abs().max().item()
    print("sparse training step: logits max|diff| %.3e (scale %.3e), loss %.5f vs oracle %.5f" % (
        err, scale, loss.item(), o_loss.item()))
    assert err < 2e-2 * scale and abs(loss.item() - o_loss.item()) < 1e-2
    for n, p in m.named_parameters():
        ref = sdr[n].grad
        e = ((p.grad.float().cpu() - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()
        assert e < 6e-2, (n, e)
