"""Finetuning the super-resolution model on the GPU: make_super_resolution_batch with the real-shaped VQ-VAE, one
finetune step on 2121-token two-image rows (positions restarting at [ROI2], clamped to the 1089-entry table) against
the CPU oracle, and rows -> file -> make_batch -> train_step -> generate.super_resolution end to end.

The model is the 2-layer d=256 configuration with a 101-piece text vocabulary (8192 + 101 + 27 = 8320 tokens), so
that the oracle's [2, 2120, 8320] logits stay cheap.  The oracle runs on the bf16-rounded weights the GPU model holds;
tolerances are those of tests/test_model_gpu.py and smoke(): logits within 2e-2 of their scale, the loss within
1e-2, per-token losses within 5e-2, gradients within 6e-2 of their own scale.  Every input is seeded."""
import random
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cogview_oracle as O
from oracle import recipes

pytestmark = pytest.mark.gpu

N_TXT = 101
VOCAB = 8192 + N_TXT + 27
MPE, MPE_FT = 1089, 2121
CFG = dict(num_layers=2, vocab_size=VOCAB, hidden_size=256, num_attention_heads=4, max_sequence_length=MPE)
FT = types.SimpleNamespace(finetune=True, max_position_embeddings=MPE, max_position_embeddings_finetune=MPE_FT)
PW = [0, 128, 256] * 3
PH = [0, 0, 0, 128, 128, 128, 256, 256, 256]


@pytest.fixture(autouse=True)
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


@pytest.fixture(scope="module")
def vq():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import vqvae
    model = vqvae.new_model()
    model.load_state_dict(recipes.vqvae_state_dict(seed=0))
    return model.cuda().eval()


def gpt(max_memory_length=0, checkpoint_activations=False, sd=None):
    from cogview_b200.model import GPT2Model
    m = GPT2Model(num_layers=CFG["num_layers"], vocab_size=VOCAB, hidden_size=CFG["hidden_size"],
                  num_attention_heads=CFG["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=MPE,
                  max_memory_length=max_memory_length, checkpoint_activations=checkpoint_activations)
    m.load_state_dict(sd if sd is not None else recipes.gpt2_state_dict(seed=41, **CFG))
    return m.cuda().bfloat16()


def texts(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [(8192 + torch.randint(0, N_TXT, (t,), generator=g)).tolist() for t in lens]


def test_builder_codes_equal_separate_img2code(vq):
    """Each row's overview codes are img2code of that image bilinearly downsampled to 256 x 256, and its patch codes
    img2code of the 256 x 256 crop at the row's [POSi], each encoded on its own."""
    from cogview_b200 import data as D
    from cogview_b200 import vqvae
    from cogview_b200.generation.sampling import get_tokenizer
    tk = get_tokenizer()
    imgs = recipes.images(2, size=512, seed=5).cuda()
    txt = texts([9, 64], seed=6)
    random.seed(7)
    rows = D.make_super_resolution_batch(vq, txt, imgs, sampling_num=3)
    assert len(rows) == 6
    for i in range(2):
        over = vqvae.img2code(vq, F.interpolate(imgs[i:i + 1], size=(256, 256), mode='bilinear')).cpu().view(-1)
        T = len(txt[i])
        for j in range(3):
            r = rows[i * 3 + j]
            assert len(r) == T + 2057
            assert torch.equal(r[T + 3:T + 1027], over)
            p = int(r[T + 1029]) - tk['[POS0]']
            patch = imgs[i:i + 1, :, PH[p]:PH[p] + 256, PW[p]:PW[p] + 256].contiguous()
            assert torch.equal(r[T + 1032:T + 2056], vqvae.img2code(vq, patch).cpu().view(-1))


def _rows(lens, seed):
    """Two-image rows with synthetic codes, padded with [PAD] to 2121 as filled_tokenized_process_fn pads them."""
    from cogview_b200 import data as D
    g = torch.Generator().manual_seed(seed)

    def encode(x):
        return torch.randint(0, 8192, (x.shape[0], 1024), generator=g)
    random.seed(seed)
    rows = D.make_super_resolution_batch(None, texts(lens, seed), torch.zeros(len(lens), 3, 512, 512),
                                         sampling_num=1, encode=encode)
    fn = D.filled_tokenized_process_fn(MPE_FT)
    items = [fn(np.concatenate((r.numpy(), -np.ones(MPE_FT - len(r), dtype=np.int64)))) for r in rows]
    return {k: np.stack([it[k] for it in items]) for k in ('text', 'loss_mask')}


@pytest.fixture(scope="module")
def oracle_step():
    """The oracle's forward, per-token losses, weighted loss and gradients for two rows of 2121 tokens (T = 64: the
    first segment's tail clamped to position 1088; T = 20: 44 [PAD] at the end, outside the loss mask)."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import data as D
    from cogview_b200.generation import sampling
    saved = sampling._TOKENIZER
    sampling._TOKENIZER = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    try:
        batch = _rows([64, 20], seed=8)
        tokens, labels, loss_mask, mask, pos = D.make_batch(batch, args=FT)
    finally:
        sampling._TOKENIZER = saved
    assert int(pos.max()) == MPE - 1 and int((pos == MPE - 1).sum()) > 2
    sd = {k: v.to(torch.bfloat16).float().requires_grad_(True)
          for k, v in recipes.gpt2_state_dict(seed=41, **CFG).items()}
    logits, _ = O.gpt2_forward(sd, CFG["num_attention_heads"], tokens, pos, mask)
    losses = O.vocab_parallel_cross_entropy(logits, labels)
    loss = O.weighted_loss(losses, tokens, loss_mask, 8192, 1.0)
    loss.backward()
    return dict(batch=(tokens, labels, loss_mask, mask, pos), logits=logits.detach(), losses=losses.detach(),
                loss=loss.item(), grads={k: v.grad for k, v in sd.items()})


@pytest.mark.parametrize("fused_loss,ckpt", [(False, False), (True, False), (False, True), (True, True)])
def test_finetune_step_matches_oracle(oracle_step, fused_loss, ckpt):
    from cogview_b200 import pretrain
    o = oracle_step
    m = gpt(checkpoint_activations=ckpt).train()
    batch = tuple(t.cuda() for t in o["batch"])
    assert batch[0].shape == (2, MPE_FT - 1)
    if fused_loss:
        loss, _, _, _ = pretrain.forward_step(batch, m, fused_loss=True)
        with torch.no_grad():
            losses, *_ = m(batch[0], batch[4], batch[3], None, None, 0, labels=batch[1])
    else:
        with torch.no_grad():
            logits, *_ = m(batch[0], batch[4], batch[3], None, None, 0)
        scale = o["logits"].abs().max().item()
        err = (logits.float().cpu() - o["logits"]).abs().max().item()
        print("logits: max|diff| %.3e, scale %.3e" % (err, scale))
        assert err < 2e-2 * scale
        losses = None
        loss, _, _, _ = pretrain.forward_step(batch, m, fused_loss=False)
    loss.backward()
    print("fused %d ckpt %d: loss %.5f oracle %.5f" % (fused_loss, ckpt, loss.item(), o["loss"]))
    assert abs(loss.item() - o["loss"]) < 1e-2
    if losses is not None:
        assert (losses.float().cpu() - o["losses"]).abs().max().item() < 5e-2
    for name in ("transformer.position_embeddings.weight", "transformer.layers.0.mlp.dense_h_to_4h.weight",
                 "word_embeddings.weight"):
        got = dict(m.named_parameters())[name].grad.float().cpu()
        ref = o["grads"][name]
        e = ((got - ref).abs().max() / ref.abs().max()).item()
        print("  %s: relative gradient error %.3e" % (name, e))
        assert e < 6e-2, (name, e)
    # every position of the table the rows use got a gradient, the clamped 1088 included
    used = torch.unique(o["batch"][4])
    assert bool((dict(m.named_parameters())["transformer.position_embeddings.weight"].grad[used.cuda()] != 0)
                .any(dim=1).all())


def test_finetune_end_to_end(vq, tok, tmp_path, monkeypatch):
    """make_super_resolution_batch -> write_tokenized_rows -> BinaryDataset -> make_batch(args=ft) -> three
    train_steps with FusedAdamW, then generate.super_resolution on the finetuned weights."""
    from cogview_b200 import data as D
    from cogview_b200 import generate, pretrain
    from cogview_b200.model import gpt2_get_params_for_weight_decay_optimization
    from cogview_b200.optim import FusedAdamW
    imgs = recipes.images(2, size=512, seed=11).cuda()
    random.seed(12)
    rows = D.make_super_resolution_batch(vq, texts([30, 64], seed=13), imgs, sampling_num=2)
    path = str(tmp_path / "sr.bin")
    D.write_tokenized_rows(path, rows, MPE_FT)
    ds = D.BinaryDataset(path, D.filled_tokenized_process_fn(MPE_FT), length_per_sample=MPE_FT)
    assert len(ds) == 4
    m = gpt().train()
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    opt = FusedAdamW(gpt2_get_params_for_weight_decay_optimization(m), lr=1e-3, weight_decay=0.01,
                     max_grad_norm=1.0)
    losses = []
    for step in range(3):
        items = [ds[(2 * step + i) % 4] for i in range(2)]
        batch = D.make_batch({k: np.stack([it[k] for it in items]) for k in ('text', 'loss_mask')}, device="cuda",
                             args=FT)
        loss, skipped, _, _, _ = pretrain.train_step(batch, m, opt, fused_loss=True)
        assert skipped == 0
        losses.append(loss.item())
    print("finetune losses", losses)
    assert all(np.isfinite(losses))
    changed = [n for n, p in m.named_parameters() if not torch.equal(p.detach(), before[n])]
    assert "transformer.position_embeddings.weight" in changed and "word_embeddings.weight" in changed
    assert len(changed) == len(before)

    sr = gpt(max_memory_length=1345, sd=m.state_dict()).eval()
    sr.transformer.mems_mode = "kv"
    seq = torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['super-resolution'],
                                            [texts([6], seed=14)[0], rows[0][33:1057].tolist()], tokenizer=tok),
                       dtype=torch.long, device="cuda")

    class A:
        temperature, top_k, top_p, is_sparse = 1.0, 1, 0.0, 0
        img_tokenizer_num_tokens = 8192

    torch.manual_seed(0)
    codes, out = generate.super_resolution(sr, vq, A, seq)
    assert codes.shape == (1, 4096) and out.shape == (1, 3, 512, 512)
    assert int(codes.min()) >= 0 and int(codes.max()) < 8192 and bool(torch.isfinite(out).all())
