"""Attention-probability dropout of sparse TRAINING attention (is_sparse = 1; the reference applies attention_dropout to
the joint pivot + window probabilities, mpu/sparse_transformer.py:150, :719-721) — cv_attn_sparse_fwd /
cv_attn_sparse_bwd with dropout_p > 0.  As for the dense sites (tests/test_dropout_gpu.py) bitwise parity with torch's
generator is not defined; these tests pin the semantics: the keep statistics, mask replay under activation
checkpointing, and a model step against the oracle run with the kernels' own keep bits (2e-2 of the logit scale, 6e-2 of
each weight gradient's scale).  The kernels with dropout are bounded element by element against the same keep bits in
tests/test_attention_sparse_gpu.py."""
import functools
import random

import pytest
import torch

from oracle import cogview_oracle as O
from oracle import recipes
import sparse_dropout_ref as R

pytestmark = pytest.mark.gpu
P = 0.1


def _pivots(b, s, n_piv, txt_n, seed):
    random.seed(seed)
    return torch.stack([
        torch.cat((torch.arange(0, txt_n[i]),
                   torch.tensor(random.sample(range(txt_n[i], s), n_piv - txt_n[i]), dtype=torch.long)))
        for i in range(b)])


def _rmask(s, w, times):
    g = s // w
    tmp = torch.ones((g - times + 1, w, w))
    tmp = torch.tril(1 - torch.block_diag(*tmp))
    return torch.nn.functional.pad(tmp, (0, (times - 1) * w, (times - 1) * w, 0))


def test_sparse_dropout_mask_statistics():
    """Keep bits over the visible pairs behave like independent Bernoulli(1 - p) draws: keep rate on band keys and on pivot
    slots, no correlation between adjacent keys, adjacent queries, two heads, or pivot slot p and band key p (the same
    step of the same LCG stream, seeded by different Philox counters)."""
    from cogview_b200 import ops
    b, heads, s, w, times, n_piv = 1, 2, 4096, 128, 6, 768
    pivot_idx = _pivots(b, s, n_piv, (100,), seed=5)
    x = torch.zeros((b, s, heads * 64), dtype=torch.bfloat16, device="cuda")
    _, mask = ops.attn_sparse_fwd(x, x, x, heads, pivot_idx.cuda(), w, times, dropout=(P, 4321, 11))
    fwd, _ = R.decode_keep(mask, b, heads, s, n_piv, w, times)
    nkb = s // 128
    vis = R.visible(s, n_piv, w, times, pivot_idx)[0]
    band_vis, piv_vis = vis[:, :s], vis[:, nkb * 128:nkb * 128 + n_piv]
    k0 = fwd[0, 0].float()
    band, piv = k0[:, :s], k0[:, nkb * 128:nkb * 128 + n_piv]
    for name, vals in (("band keys", band[band_vis]), ("pivot slots", piv[piv_vis])):
        rate, n = vals.mean().item(), vals.numel()
        print("keep rate over visible (query, %s) pairs: %.5f (expected %.5f, n = %d)" % (name, rate, 1 - P, n))
        assert abs(rate - (1 - P)) < 5 * (P * (1 - P) / n) ** 0.5

    def corr(a, b_):
        a = a - a.mean(); b_ = b_ - b_.mean()
        return (a * b_).mean().item() / (a.std().item() * b_.std().item() + 1e-12)
    pairs = {
        "adjacent keys": (band[:, 1:], band[:, :-1], band_vis[:, 1:] & band_vis[:, :-1]),
        "adjacent queries": (band[1:], band[:-1], band_vis[1:] & band_vis[:-1]),
        "two heads": (k0[:, :s], fwd[0, 1, :, :s].float(), band_vis),
        # few pairs are visible together (pivot p needs position < band start): compare every generated decision
        "pivot slot p / band key p": (piv, band[:, :n_piv], (piv >= 0) & (band[:, :n_piv] >= 0)),
    }
    for name, (a, c, m) in pairs.items():
        n = m.sum().item()
        r = corr(a[m], c[m])
        print("correlation, %s: %.4f (bound %.4f, n = %d)" % (name, r, 5 / n ** 0.5, n))
        assert n > 1000 and abs(r) < 5 / n ** 0.5, name


def _sparse_layer_and_input(b=2, s=256, w=64, times=2, n_piv=48):
    from cogview_b200.mpu.sparse_transformer import GPT2ParallelTransformerLayer, SparseSpec, unscaled_init_method
    torch.manual_seed(7)
    layer = GPT2ParallelTransformerLayer(256, 4, 0.1, 0.1, 1e-5, unscaled_init_method(0.02), query_window=w,
                                         key_window_times=times).cuda().bfloat16().train()
    x = torch.randn((b * s, 256), device="cuda")
    spec = SparseSpec(_pivots(b, s, n_piv, (20, 0), seed=3).cuda(), w, times)
    return layer, x, spec


def test_sparse_layer_forward_replays_dropout_under_checkpointing():
    """The no-grad pass of mpu.checkpoint and the autograd recomputation draw the same three sites per layer."""
    from cogview_b200 import ops
    from cogview_b200.mpu import random as mrandom
    layer, x, spec = _sparse_layer_and_input()
    am = ops.absmax(x)
    mrandom.set_dropout_site_counter(50)
    with torch.no_grad():
        out0, _ = layer.fused_forward(x, am, 2, 256, spec)
    mrandom.set_dropout_site_counter(50)
    xg = x.clone().requires_grad_(True)
    out1, _ = layer.fused_forward(xg, am, 2, 256, spec)
    assert torch.equal(out0, out1.detach())
    mrandom.set_dropout_site_counter(60)
    with torch.no_grad():
        out2, _ = layer.fused_forward(x, am, 2, 256, spec)
    assert not torch.equal(out0, out2)
    out1.backward(torch.randn_like(out1))
    assert torch.isfinite(xg.grad).all()


def _sparse_train_step(site_counter, attn_p=0.1, out_p=0.1, emb_p=0.1, seed=4321, sd=None):
    from cogview_b200 import mpu
    from cogview_b200.model import GPT2Model
    from cogview_b200.mpu import random as mrandom
    cfg = dict(num_layers=2, vocab_size=58240, hidden_size=256, num_attention_heads=4, max_sequence_length=256)
    s, w, times, n_piv = 256, 64, 2, 48
    torch.manual_seed(seed)
    mrandom.set_dropout_site_counter(site_counter)
    m = GPT2Model(num_layers=2, vocab_size=cfg["vocab_size"], hidden_size=256, num_attention_heads=4,
                  embedding_dropout_prob=emb_p, attention_dropout_prob=attn_p, output_dropout_prob=out_p,
                  max_sequence_length=s, max_memory_length=0, checkpoint_activations=True, checkpoint_num_layers=1,
                  query_window=w, key_window_times=times, num_pivot=n_piv)
    m.load_state_dict(sd if sd is not None else recipes.gpt2_state_dict(seed=21, **cfg))
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
    return m, logits, loss, (tokens, labels, pos, img)


def test_sparse_model_training_with_dropout_is_reproducible_and_checkpoint_safe():
    m0, _, l0, _ = _sparse_train_step(100)
    g0 = {n: p.grad.float().clone() for n, p in m0.named_parameters()}
    m1, _, l1, _ = _sparse_train_step(100)
    _, _, l2, _ = _sparse_train_step(500)
    print("sparse training with dropout 0.1: loss %.5f, repeat %.5f, other sites %.5f" % (l0.item(), l1.item(), l2.item()))
    assert l0.item() == l1.item()
    assert all(torch.equal(g0[n], p.grad.float()) for n, p in m1.named_parameters())
    assert l2.item() != l0.item()
    assert torch.isfinite(l0) and all(torch.isfinite(g).all() for g in g0.values())


def test_sparse_model_with_attention_dropout_matches_oracle(monkeypatch):
    """test_model_sparse_training_step_matches_oracle with attention_dropout_prob = 0.1: the oracle applies each layer's
    keep mask, regenerated from that layer's (seed, site) — three sites per layer, the first is the attention's."""
    from cogview_b200 import ops
    from cogview_b200.mpu.sparse_transformer import GPT2ParallelTransformer
    cfg = dict(num_layers=2, vocab_size=58240, hidden_size=256, num_attention_heads=4, max_sequence_length=256)
    s, w, times, n_piv, c0 = 256, 64, 2, 48, 1000
    sd32 = recipes.gpt2_state_dict(seed=21, **cfg)
    m, logits, loss, (tokens, labels, pos, img) = _sparse_train_step(c0, attn_p=P, out_p=0.0, emb_p=0.0, sd=sd32)
    seed = torch.initial_seed()
    random.seed(77)
    img_all = [img[i].nonzero(as_tuple=False).view(-1) for i in range(2)]
    txt_all = [(~img)[i].nonzero(as_tuple=False).view(-1) for i in range(2)]
    pivots = [GPT2ParallelTransformer.sample_pivot_idx(img_all, txt_all, n_piv) for _ in range(2)]
    zeros = torch.zeros((2, s, 256), dtype=torch.bfloat16, device="cuda")
    keeps = []
    for li in range(2):
        _, mask = ops.attn_sparse_fwd(zeros, zeros, zeros, 4, pivots[li].cuda(), w, times,
                                      dropout=(P, seed, c0 + 3 * li + 1))
        fwd, _ = R.decode_keep(mask, 2, 4, s, n_piv, w, times)
        keeps.append(R.to_reference_layout(fwd, s, n_piv, w, times))
    sdr = {k: v.to(torch.bfloat16).float().requires_grad_(True) for k, v in sd32.items()}
    rm = _rmask(s, w, times)
    x = torch.nn.functional.embedding(tokens, sdr["word_embeddings.weight"]) + \
        torch.nn.functional.embedding(pos, sdr["transformer.position_embeddings.weight"])
    for li in range(2):
        pam = rm.expand(2, s, s).gather(dim=-1, index=pivots[li].unsqueeze(1).expand(2, s, n_piv))
        monkeypatch.setattr(O, "sparse_attention", functools.partial(R.sparse_attention_keep, keep=keeps[li],
                                                                     dropout_p=P))
        x = O.transformer_layer(sdr, li, x, pam, 4, is_sparse=1, pivot_idx=pivots[li], query_window=w,
                                key_window_times=times)
    monkeypatch.undo()
    xf = O.layernorm_absmax(x, sdr["transformer.final_layernorm.weight"], sdr["transformer.final_layernorm.bias"])
    o_logits = torch.nn.functional.linear(xf, sdr["word_embeddings.weight"])
    o_loss = O.vocab_parallel_cross_entropy(o_logits, labels).mean()
    o_loss.backward()
    scale = o_logits.abs().max().item()
    err = (logits.float().cpu() - o_logits.detach()).abs().max().item()
    print("sparse training step, attention dropout 0.1: logits max|diff| %.3e (scale %.3e), loss %.5f vs oracle %.5f" % (
        err, scale, loss.item(), o_loss.item()))
    assert err < 2e-2 * scale and abs(loss.item() - o_loss.item()) < 1e-2
    for n, p in m.named_parameters():
        ref = sdr[n].grad
        e = ((p.grad.float().cpu() - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()
        assert e < 6e-2, (n, e)
