"""The fused vocabulary cross-entropy (cv_vocab_xent_fwd / cv_vocab_xent_dlogits, _VocabXentFn,
GPT2Model.forward(..., labels=), pretrain.train_step(..., fused_loss=True)) against float64, the logits route
(_LogitsFn + mpu.vocab_parallel_cross_entropy), the CPU oracle and the reference's golden values."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import cogview_oracle as O
from oracle import recipes

pytestmark = pytest.mark.gpu

CFG = recipes.CONFIG1
V4B = 58240


def _operands(M, K, V, logit_std, seed):
    """bf16 H [M, K], W [V, K] with logits of standard deviation ~logit_std, targets covering 0 and V - 1."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn((V, K), generator=g, device="cuda") * 0.05).to(torch.bfloat16)
    h = (torch.randn((M, K), generator=g, device="cuda") * (logit_std / (0.05 * K ** 0.5))).to(torch.bfloat16)
    t = torch.randint(0, V, (M,), generator=g, device="cuda")
    t[0] = 0
    t[-1] = V - 1
    if M > 2:
        t[1] = V - 1
    return h, w, t


def _lse64(h, w, chunk=4096):
    """float64 row log-sum-exp of h @ w^T and the logits' target values, a few thousand columns at a time."""
    h64 = h.double()
    mx = torch.full((h.shape[0],), -float("inf"), dtype=torch.float64, device=h.device)
    s = torch.zeros_like(mx)
    for v0 in range(0, w.shape[0], chunk):
        z = h64 @ w[v0:v0 + chunk].double().t()
        nm = torch.maximum(mx, z.max(1).values)
        s = s * torch.exp(mx - nm) + torch.exp(z - nm[:, None]).sum(1)
        mx = nm
    return mx + torch.log(s)


@pytest.mark.parametrize("M", [1, 127, 128, 1000, 4352])
@pytest.mark.parametrize("K,V", [(256, V4B), (320, V4B), (2560, V4B), (256, 1000), (320, 4321)])
def test_forward_kernel_matches_float64(M, K, V):
    from cogview_b200 import ops
    h, w, t = _operands(M, K, V, 60.0, seed=M + K + V)
    loss, lse = ops.vocab_xent_fwd(h, w, t)
    want_lse = _lse64(h, w)
    want_loss = want_lse - (h.double() * w[t].double()).sum(1)
    zmax = float((h.double() @ w[:4096].double().t()).abs().max())
    assert zmax > 100, zmax                          # the logits span hundreds
    for got, want in ((loss, want_loss), (lse, want_lse)):
        err = (got.double() - want).abs()
        assert bool(torch.isfinite(got).all())
        assert bool((err <= 1e-3 + 1e-4 * want.abs()).all()), float(err.max())


def test_forward_target_outside_the_vocabulary_gives_nan():
    from cogview_b200 import ops
    h, w, t = _operands(130, 256, 1000, 5.0, seed=3)
    t[5], t[129] = -1, 1000
    loss, lse = ops.vocab_xent_fwd(h, w, t)
    assert bool(torch.isnan(loss[5])) and bool(torch.isnan(loss[129]))
    keep = torch.ones(130, dtype=torch.bool, device="cuda")
    keep[5] = keep[129] = False
    assert bool(torch.isfinite(loss[keep]).all()) and bool(torch.isfinite(lse).all())


@pytest.mark.parametrize("M,K,V,v_begin,v_end", [
    (300, 320, 5000, 100, 1234),        # starts and ends mid-tile
    (300, 320, 5000, 0, 5000),
    (129, 256, 5000, 4000, 4999),
    (129, 256, 5000, 257, 258),         # one column
    (1000, 2560, V4B, 30000, 30000 + 3 * 256 + 77),
])
def test_dlogits_kernel_matches_float64(M, K, V, v_begin, v_end):
    from cogview_b200 import ops
    h, w, t = _operands(M, K, V, 8.0, seed=v_begin + M)
    # some targets inside the window, the rest anywhere
    t[2::3] = torch.randint(v_begin, v_end, (t[2::3].numel(),), device="cuda")
    g = torch.randn(M, device="cuda")
    g[::5] = 0.0
    _, lse = ops.vocab_xent_fwd(h, w, t)
    n = v_end - v_begin
    ldd = (n + 7) // 8 * 8 + 8
    buf = torch.full((M + 3, ldd), float("nan"), dtype=torch.bfloat16, device="cuda")
    d = ops.vocab_xent_dlogits(h, w, t, lse, g, v_begin, v_end, out=buf[:M])
    assert d.shape == (M, n)
    z = h.double() @ w[v_begin:v_end].double().t()
    p = torch.exp(z - _lse64(h, w)[:, None])
    onehot = torch.zeros_like(p)
    inwin = (t >= v_begin) & (t < v_end)
    onehot[inwin.nonzero().view(-1), (t[inwin] - v_begin)] = 1.0
    want = g.double()[:, None] * (p - onehot)
    got = d.double()
    err = (got - want).abs()
    tol = 2 ** -8 * want.abs() + 1e-3 * g.double().abs()[:, None] * p + 1e-30
    assert bool((err <= tol).all()), float((err / tol).max())
    assert bool((got[::5] == 0).all())                              # rows with grad_loss = 0 are exactly zero
    assert bool(torch.isnan(buf[:M, n:].float()).all())              # columns past the window: not written
    assert bool(torch.isnan(buf[M:].float()).all())                  # rows past M: not written


def _leaves(h, w):
    return h.clone().requires_grad_(True), w.clone().requires_grad_(True)


def _old_stage(hh, ww, t, g):
    """The logits route on the leaves hh, ww: (losses, dH, dW)."""
    from cogview_b200 import mpu
    from cogview_b200.model.gpt2_modeling import _LogitsFn
    hh.grad = ww.grad = None
    losses = mpu.vocab_parallel_cross_entropy(_LogitsFn.apply(hh, ww).float(), t)
    (losses * g).sum().backward()
    return losses.detach(), hh.grad, ww.grad


def _new_stage(hh, ww, t, g, budget):
    from cogview_b200.model.gpt2_modeling import _VocabXentFn
    hh.grad = ww.grad = None
    losses = _VocabXentFn.apply(hh, ww, t, budget)
    (losses * g).sum().backward()
    return losses.detach(), hh.grad, ww.grad


@pytest.mark.parametrize("budget", ["many", "one"])
def test_loss_stage_matches_the_logits_route(budget):
    from cogview_b200 import ops
    M, K, V = 1100, 256, V4B
    h, w, t = _operands(M, K, V, 4.0, seed=11)
    g = torch.rand(M, device="cuda") / M
    nbytes = M * 2 * 2048 if budget == "many" else None
    chunks = ops.xent_chunks(M, V, nbytes)
    assert (len(chunks) > 20 and chunks[-1][1] - chunks[-1][0] < 2048) if budget == "many" else len(chunks) == 1
    l0, dh0, dw0 = _old_stage(*_leaves(h, w), t, g)
    l1, dh1, dw1 = _new_stage(*_leaves(h, w), t, g, nbytes)
    assert dh1.dtype == dh0.dtype and dw1.dtype == dw0.dtype
    el = (l1 - l0).abs().max().item()
    eh = ((dh1.float() - dh0.float()).abs().max() / dh0.float().abs().max()).item()
    ew = ((dw1.float() - dw0.float()).abs().max() / dw0.float().abs().max()).item()
    print("loss stage (%d chunks): loss %.2e, dH %.2e, dW %.2e of scale" % (len(chunks), el, eh, ew))
    assert el < 1e-4 and eh < 1e-2 and ew < 1e-2


def test_repeats_are_bit_equal():
    from cogview_b200 import ops
    M, K, V = 777, 320, V4B
    h, w, t = _operands(M, K, V, 20.0, seed=5)
    g = torch.randn(M, device="cuda")
    budget = M * 2 * 4096
    outs = []
    for _ in range(2):
        loss, lse = ops.vocab_xent_fwd(h, w, t)
        dh, dw = ops.vocab_xent_bwd(h, w, t, lse, g, budget)
        outs.append((loss, lse, dh, dw))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_loss_stage_memory():
    """The rise of max_memory_allocated over forward + backward of the loss stage at M = 8192, K = 256, V = 58240.
    Every route returns the [V, K] weight gradient; beyond that the fused route holds at most one dlogits chunk and
    a few [M, K] buffers, where the logits route holds the [M, V] fp32 logits (1.9 GB) and more."""
    from cogview_b200 import ops
    M, K, V = 8192, 256, V4B
    h, w, t = _operands(M, K, V, 4.0, seed=8)
    g = torch.full((M,), 1.0 / M, device="cuda")

    hh, ww = _leaves(h, w)

    def rise(fn):
        hh.grad = ww.grad = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = fn()
        torch.cuda.synchronize()
        r = torch.cuda.max_memory_allocated() - base
        del out
        return r

    old = rise(lambda: _old_stage(hh, ww, t, g))
    new = rise(lambda: _new_stage(hh, ww, t, g, None))
    dw_bytes = V * K * 2
    print("loss stage peak rise at M=%d: logits route %.1f MB, fused route %.1f MB (of which dW %.1f MB)" % (
        M, old / 1e6, new / 1e6, dw_bytes / 1e6))
    assert new - dw_bytes < ops.XENT_CHUNK_BYTES + 4 * M * K * 4
    assert old > M * V * 4 > new


def _build(checkpoint_activations=False):
    from cogview_b200.model import GPT2Model
    m = GPT2Model(num_layers=CFG["num_layers"], vocab_size=CFG["vocab_size"], hidden_size=CFG["hidden_size"],
                  num_attention_heads=CFG["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0,
                  max_sequence_length=CFG["max_sequence_length"], max_memory_length=0,
                  checkpoint_activations=checkpoint_activations)
    m.load_state_dict(recipes.gpt2_state_dict(**CFG))
    return m.cuda().bfloat16()


@pytest.fixture(scope="module")
def data(golden_dir):
    g = np.load(os.path.join(golden_dir, "gpt2_config1.npz"))
    tf = torch.from_numpy(g["tokens_full"])
    tokens, labels = tf[:, :-1].contiguous(), tf[:, 1:].contiguous()
    s = tokens.shape[1]
    pos = torch.arange(s).unsqueeze(0).expand_as(tokens).contiguous()
    sd = {k: v.to(torch.bfloat16).float() for k, v in recipes.gpt2_state_dict(**CFG).items()}
    return dict(g=g, tokens=tokens, labels=labels, pos=pos, sd=sd, s=s)


@pytest.mark.parametrize("ckpt", [False, True])
def test_model_training_step_with_labels_matches_oracle_and_golden(data, ckpt):
    """forward(..., labels=) + the reference's loss weighting (pretrain_gpt2.py:305-321) + backward, with the
    tolerances of the logits route's own test against the oracle and the golden gradient norms."""
    m = _build(ckpt).train()
    g, s = data["g"], data["s"]
    tokens, labels = data["tokens"].cuda(), data["labels"].cuda()
    mask = torch.tril(torch.ones((1, 1, s, s), device="cuda"))
    losses, *_ = m(tokens, data["pos"].cuda(), mask, None, None, 0, labels=labels)
    assert losses.shape == tokens.shape and losses.dtype == torch.float32
    txt_scale = float(g["txt_loss_scale"])
    lm = torch.ones_like(tokens, dtype=torch.float)
    lm[tokens >= recipes.IMG_VOCAB] *= txt_scale
    loss = torch.sum(losses.view(-1) * lm.view(-1)) / lm.sum()
    loss.backward()
    sdr = {k: v.clone().requires_grad_(True) for k, v in data["sd"].items()}
    o_logits, _ = O.gpt2_forward(sdr, CFG["num_attention_heads"], data["tokens"], data["pos"],
                                 torch.tril(torch.ones((1, 1, s, s))))
    o_losses = O.vocab_parallel_cross_entropy(o_logits, data["labels"])
    o_loss = O.weighted_loss(o_losses, data["tokens"], torch.ones_like(data["tokens"], dtype=torch.float),
                             recipes.IMG_VOCAB, txt_scale)
    o_loss.backward()
    print("fused loss %.5f oracle %.5f reference %.5f" % (loss.item(), o_loss.item(), float(g["loss"])))
    assert (losses.float().cpu() - o_losses.detach()).abs().max().item() < 5e-2
    assert abs(loss.item() - o_loss.item()) < 1e-2
    assert abs(loss.item() - float(g["loss"])) < 2e-2
    names = [str(n) for n in g["grad_names"]]
    for n, p in m.named_parameters():
        assert p.grad is not None, n
        ref = sdr[n].grad
        e = ((p.grad.float().cpu() - ref).abs().max() / ref.abs().max().clamp_min(1e-12)).item()
        assert e < 6e-2, (n, e)
        gn = float(p.grad.float().norm())
        rn = float(g["grad_norms"][names.index(n)])
        assert abs(gn - rn) < 5e-2 * rn, (n, gn, rn)


def test_labels_equal_the_logits_route_and_evaluate_without_autograd(data):
    from cogview_b200 import mpu
    m = _build().train()
    s = data["s"]
    args = (data["tokens"].cuda(), data["pos"].cuda(), torch.tril(torch.ones((1, 1, s, s), device="cuda")), None,
            None, 0)
    labels = data["labels"].cuda()
    logits, *_ = m(*args)
    want = mpu.vocab_parallel_cross_entropy(logits.contiguous().float(), labels).detach()
    got, *_ = m(*args, labels=labels)
    with torch.no_grad():
        ev, *_ = m(*args, labels=labels)
    assert not ev.requires_grad and got.requires_grad
    print("labels= vs logits route %.2e, no_grad vs autograd %.2e" % ((got - want).abs().max().item(),
                                                                      (ev - got).abs().max().item()))
    assert (got.detach() - want).abs().max().item() < 1e-4
    assert (ev - got.detach()).abs().max().item() < 1e-4


def test_train_step_fused_loss_tracks_the_logits_route():
    from cogview_b200 import pretrain
    from cogview_b200.generation.sampling import get_masks_and_position_ids
    from cogview_b200.model import gpt2_get_params_for_weight_decay_optimization
    from cogview_b200.optim import FusedAdamW
    tf = recipes.text_image_tokens(2, 32, 97, seed=9).cuda()
    tokens, labels = tf[:, :-1].contiguous(), tf[:, 1:].contiguous()
    mask, loss_mask, pos = get_masks_and_position_ids(tokens)
    batch = (tokens, labels, loss_mask, mask, pos)
    curves = []
    for fused in (False, True):
        m = _build().train()
        groups = gpt2_get_params_for_weight_decay_optimization(m)
        opt = FusedAdamW(groups, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_grad_norm=1.0)
        losses = []
        for _ in range(4):
            loss, skipped, *_ = pretrain.train_step(batch, m, opt, txt_loss_scale=0.5, fused_loss=fused)
            assert skipped == 0
            losses.append(loss.item())
        curves.append(losses)
    print("train_step losses: logits route %s, fused %s" % tuple(curves))
    assert curves[0][-1] < curves[0][0]
    for a, b in zip(*curves):
        assert abs(a - b) < 2e-2 * abs(a)


def test_sparse_training_step_with_labels_matches_the_logits_route():
    from cogview_b200 import mpu
    from cogview_b200.model import GPT2Model
    cfg = dict(num_layers=2, vocab_size=V4B, hidden_size=256, num_attention_heads=4, max_sequence_length=256)
    s, w, times, n_piv = 256, 64, 2, 48
    sd32 = recipes.gpt2_state_dict(seed=21, **cfg)
    tokens = recipes.text_image_tokens(2, 32, s - 32, seed=3)
    labels = torch.roll(tokens, -1, dims=1).cuda()
    pos = torch.arange(s).unsqueeze(0).expand(2, -1).contiguous().cuda()
    img = tokens < recipes.IMG_VOCAB
    runs = []
    for fused in (False, True):
        m = GPT2Model(num_layers=2, vocab_size=V4B, hidden_size=256, num_attention_heads=4,
                      embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                      max_sequence_length=s, max_memory_length=0, checkpoint_activations=True,
                      checkpoint_num_layers=1, query_window=w, key_window_times=times, num_pivot=n_piv)
        m.load_state_dict(sd32)
        m = m.cuda().bfloat16().train()
        random.seed(77)
        args = (tokens.cuda(), pos, torch.tril(torch.ones((1, 1, s, s), device="cuda")), (~img).cuda(), img.cuda(), 1)
        if fused:
            losses, *_ = m(*args, labels=labels)
        else:
            logits, *_ = m(*args)
            losses = mpu.vocab_parallel_cross_entropy(logits.contiguous().float(), labels)
        losses.mean().backward()
        runs.append((losses.detach(), {n: p.grad.float() for n, p in m.named_parameters()}))
    (l0, g0), (l1, g1) = runs
    assert (l1 - l0).abs().max().item() < 1e-3
    for n in g0:
        e = ((g1[n] - g0[n]).abs().max() / g0[n].abs().max().clamp_min(1e-12)).item()
        assert e < 1e-2, (n, e)


def test_argument_errors():
    from cogview_b200 import _lib, ops
    lib = _lib.lib()
    h, w, t = _operands(64, 256, 1000, 1.0, seed=1)
    loss = torch.empty(64, device="cuda")
    lse = torch.empty(64, device="cuda")
    g = torch.ones(64, device="cuda")
    d = torch.empty((64, 1000), dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(lib.cv_vocab_xent_workspace_bytes(64, 1000) // 4, device="cuda")
    s = _lib.stream_ptr()
    P = _lib.ptr

    def fwd(**kw):
        a = dict(H=P(h), ldh=256, W=P(w), ldw=256, target=P(t), loss=P(loss), lse=P(lse), ws=P(ws), M=64, K=256,
                 V=1000)
        a.update(kw)
        return lib.cv_vocab_xent_fwd(*a.values(), s)

    def dl(**kw):
        a = dict(H=P(h), ldh=256, W=P(w), ldw=256, target=P(t), lse=P(lse), g=P(g), D=P(d), ldd=1000, M=64, K=256,
                 v0=0, v1=1000)
        a.update(kw)
        return lib.cv_vocab_xent_dlogits(*a.values(), s)

    assert fwd() == 0 and dl() == 0
    for rc in (fwd(H=0), fwd(loss=0), fwd(ws=0), fwd(ldh=100), fwd(ldw=255), fwd(M=0), fwd(V=0),
               dl(W=0), dl(lse=0), dl(g=0), dl(D=0), dl(ldh=12), dl(ldd=999), dl(ldd=998), dl(v0=500, v1=500),
               dl(v0=600, v1=500), dl(v0=-1)):
        assert rc < 0
        assert lib.cv_last_error()
    with pytest.raises(_lib.CogViewB200Error, match="ldd"):
        _lib.check(dl(ldd=999), "cv_vocab_xent_dlogits")
    m = _build().eval()
    tok = torch.zeros((1, 8), dtype=torch.long, device="cuda")
    pos = torch.arange(8, device="cuda").view(1, 8)
    with torch.no_grad(), pytest.raises(ValueError):
        m(tok, pos, torch.tril(torch.ones((1, 1, 8, 8), device="cuda")), None, None, 0, labels=tok,
          logits_last_only=True)
    assert ops.xent_chunks(64, 1000) == [(0, 1000)]
