"""The kernel paths taken at hidden sizes that are not multiples of 256 (hidden = 64 * heads with heads % 4 != 0: 192,
320, 384, 640, ...) and above 2560, checked against float64 CPU references on the bf16-rounded inputs.

The library picks kernels by hidden size in several places:
  * LayerNorm forward: the register kernel for rows without a residual and cols <= 2560, the shared-memory staged
    kernel otherwise (csrc/layernorm.cu cv_layernorm_absmax_fwd);
  * LayerNorm backward: the fused kernel for cols % 256 == 0 and cols <= 4096, else ln_bwd_dx_kernel +
    ln_bwd_param_kernel + ln_bwd_finalize_kernel;
  * layer backward: bias gradients from the fused LayerNorm backward's column sums, or from cv_colsum_bf16.

Errors are checked per row (per 128 x 128 block for GEMM outputs) against that row's (block's) scale, so a wrong tail
row or tile cannot hide behind a large value elsewhere.  Tolerances as in test_kernels_gpu.py: 2e-2 of the scale for
bf16 outputs, 1e-4 for fp32 outputs.  Every input is seeded."""
import pytest
import torch

from oracle import cogview_oracle as O
from oracle import recipes

pytestmark = pytest.mark.gpu
P = 0.1
F32, BF16 = torch.float32, torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


def bf(x):
    return x.to(torch.bfloat16)


def tol(dtype):
    return 2e-2 if dtype == torch.bfloat16 else 1e-4


def row_err(got, want, floor=0.0):
    """max over rows of max|got - want| / (scale of the row); the last dimension is the row.  floor > 0 raises every
    row's scale to at least that fraction of the whole tensor's scale (for gradients, whose rows can be near zero)."""
    got = got.detach().double().cpu().reshape(-1, got.shape[-1])
    want = want.detach().double().cpu().reshape(-1, want.shape[-1])
    scale = want.abs().amax(-1).clamp_min(floor * want.abs().max().item()).clamp_min(1e-300)
    return ((got - want).abs().amax(-1) / scale).max().item()


def block_err(got, want, blk=128):
    """max over 128 x 128 blocks of max|got - want| / max|want| of the block."""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    M, N = want.shape
    mb, nb = -(-M // blk), -(-N // blk)

    def blocks(t):
        p = torch.zeros((mb * blk, nb * blk), dtype=torch.float64)
        p[:M, :N] = t
        return p.view(mb, blk, nb, blk).amax(dim=(1, 3))
    return (blocks((got - want).abs()) / blocks(want.abs()).clamp_min(1e-300)).max().item()


# ----------------------------------------------------------------------------------------------------
# LayerNorm forward: every dispatch branch
# ----------------------------------------------------------------------------------------------------
def _ln_data(rows, cols, x_dtype, seed):
    g = torch.Generator().manual_seed(seed)
    scale = 10.0 ** (torch.rand((rows, 1), generator=g) * 2 - 1)          # rows of different scale (0.1 .. 10)
    x = (torch.randn((rows, cols), generator=g) + torch.randn((rows, 1), generator=g)) * scale
    x = x.to(x_dtype)
    gamma, beta = bf(1 + 0.1 * torch.randn(cols, generator=g)), bf(0.1 * torch.randn(cols, generator=g))
    return g, x, gamma, beta


def _ln_stats64(x):
    x = x.double()
    c = x.abs().max() / 8
    var = x.var(-1, unbiased=False)
    return x.mean(-1), 1.0 / torch.sqrt(var + O.LN_EPS * c * c)


# (x dtype, out dtype, residual): every combination cv_layernorm_absmax_fwd accepts
LN_FWD_COMBOS = [(F32, BF16, False), (BF16, F32, True), (BF16, BF16, False), (F32, F32, False), (F32, F32, True)]


@pytest.mark.parametrize("combo", LN_FWD_COMBOS, ids=lambda c: "%s-%s-%s" % (str(c[0])[6:], str(c[1])[6:],
                                                                             "res" if c[2] else "nores"))
@pytest.mark.parametrize("cols", [196, 320, 1000, 2560, 3072, 4096])
def test_layernorm_fwd_every_branch(ops, cols, combo):
    """cols <= 2560 without a residual: the register kernel (196, 320, 1000 end in a partial 128-column group);
    with a residual or cols > 2560: the staged kernel."""
    x_dtype, out_dtype, res = combo
    for rows in (1, 7, 300):
        g, x, gamma, beta = _ln_data(rows, cols, x_dtype, seed=rows * 7919 + cols)
        residual = torch.randn((rows, cols), generator=g) if res else None
        am = ops.absmax(x.cuda())
        amo = torch.zeros(1, device="cuda")
        out, mean, rstd = ops.layernorm_absmax_fwd(x.cuda(), am, gamma.cuda(), beta.cuda(), O.LN_EPS,
                                                   residual=residual.cuda() if res else None, out_dtype=out_dtype,
                                                   absmax_out=amo, save_stats=True)
        ref = O.layernorm_absmax(x.double(), gamma.double(), beta.double())
        if res:
            ref = ref + residual.double()
        mean64, rstd64 = _ln_stats64(x)
        e = row_err(out, ref)
        assert e < tol(out_dtype), (rows, "out", e)
        xmax = x.double().abs().amax(-1)
        assert ((mean.cpu().double() - mean64).abs() / xmax).max().item() < 1e-4, (rows, "mean")
        assert ((rstd.cpu().double() - rstd64).abs() / rstd64).max().item() < 1e-4, (rows, "rstd")
        # abs-max of the stored values, exactly (the next LayerNorm's scale)
        assert amo.item() == out.float().abs().max().item(), rows


# ----------------------------------------------------------------------------------------------------
# LayerNorm backward: fused and unfused paths, dropout on both
# ----------------------------------------------------------------------------------------------------
# (x dtype, dy dtype, dx dtype): every combination cv_layernorm_absmax_bwd accepts
LN_BWD_COMBOS = [(BF16, F32, BF16), (F32, BF16, F32), (F32, F32, F32), (BF16, BF16, BF16)]


@pytest.mark.parametrize("combo", LN_BWD_COMBOS, ids=lambda c: "-".join(str(t)[6:] for t in c))
@pytest.mark.parametrize("cols", [256, 2560, 4096, 192, 320, 1000, 3520])
def test_layernorm_bwd_both_paths(ops, cols, combo):
    """rows 1 and 3: fewer than the fused kernel's 4 rows per step; 33: a ragged split over the unfused parameter
    kernel's 32 row splits; 1000: more rows than the grid.  dx against fp64 autograd of O.layernorm_absmax; with
    dropout, dx is the no-dropout dx times the keep mask of the site / (1 - p) (the mask cv_dropout_mask reports)."""
    x_dtype, dy_dtype, dx_dtype = combo
    fused = cols % 256 == 0
    for rows in (1, 3, 33, 1000):
        g, x, gamma, beta = _ln_data(rows, cols, x_dtype, seed=rows * 31 + cols)
        dy = torch.randn((rows, cols), generator=g).to(dy_dtype)
        dres = torch.randn((rows, cols), generator=g)
        xc, dyc, gc = x.cuda(), dy.cuda(), gamma.cuda()
        _, mean, rstd = ops.layernorm_absmax_fwd(xc, ops.absmax(xc), gc, beta.cuda(), O.LN_EPS, save_stats=True)
        xr = x.double().requires_grad_(True)
        gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        O.layernorm_absmax(xr, gr, br).backward(dy.double())
        for with_dres in (False, True):
            dr = dres.cuda() if with_dres else None
            dx, dg, db = ops.layernorm_absmax_bwd(xc, dyc, mean, rstd, gc, dres=dr, dx_dtype=dx_dtype)
            want = xr.grad + dres.double() if with_dres else xr.grad
            e = row_err(dx, want)
            assert e < tol(dx_dtype), (rows, with_dres, "dx", e)
            assert row_err(dg[None], gr.grad[None]) < 2e-2, (rows, "dgamma")
            assert row_err(db[None], br.grad[None]) < 2e-2, (rows, "dbeta")
            if fused:
                dx2, dg2, db2, dxsum = ops.layernorm_absmax_bwd(xc, dyc, mean, rstd, gc, dres=dr, dx_dtype=dx_dtype,
                                                                want_dxsum=True)
                assert torch.equal(dx2, dx) and torch.equal(dg2, dg) and torch.equal(db2, db)
                _check_colsum(dxsum, dx)
            # dropout: the site's keep mask / (1 - p) on dx; the parameter gradients do not depend on it
            site = 11 + rows
            mask = ops.dropout_mask(rows * cols, P, 1234, site).view(rows, cols)
            r = ops.layernorm_absmax_bwd(xc, dyc, mean, rstd, gc, dres=dr, dx_dtype=dx_dtype, dropout=(P, 1234, site),
                                         want_dxsum=fused)
            dxd = r[0]
            assert torch.equal(r[1], dg) and torch.equal(r[2], db)
            assert bool((dxd[mask == 0] == 0).all()), (rows, "dropped elements must be 0")
            e = row_err(dxd, dx.double() * mask.double() / (1 - P))
            assert e < (1e-2 if dx_dtype == BF16 else 1e-6), (rows, with_dres, "dx with dropout", e)
            if fused:
                _check_colsum(r[3], dxd)


def _check_colsum(got, m):
    """got: bf16 column sums of the stored matrix m.  Each column within bf16 rounding of its own sum, plus the fp32
    accumulation error allowance of 1e-5 of its sum of magnitudes."""
    m = m.detach().double().cpu()
    want, mag = m.sum(0), m.abs().sum(0)
    err = (got.double().cpu() - want).abs()
    bad = err > 4e-3 * want.abs() + 1e-5 * mag + 1e-30
    assert not bool(bad.any()), ("column sums", bad.nonzero()[:8].view(-1).tolist(), err.max().item())


def test_unfused_layernorm_bwd_refuses_rows_beyond_the_row_cache(ops):
    """cols % 256 != 0 above 3520 columns: two fp32 rows per warp no longer fit in shared memory; the call must fail
    on the host with a clear message."""
    from cogview_b200._lib import CogViewB200Error
    rows, cols = 8, 4160
    x = torch.zeros((rows, cols), device="cuda")
    st = torch.ones(rows, device="cuda")
    gamma = torch.ones(cols, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(CogViewB200Error, match="row cache"):
        ops.layernorm_absmax_bwd(x, x, st, st, gamma)


# ----------------------------------------------------------------------------------------------------
# column sums (bias gradients when h % 256 != 0)
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [2, 192, 1000, 7680])
@pytest.mark.parametrize("rows", [1, 31, 33, 4352])
def test_colsum(ops, rows, cols):
    g = torch.Generator().manual_seed(rows * 13 + cols)
    m = bf(torch.randn((rows, cols), generator=g) * (1 + torch.rand(cols, generator=g) * 4))
    assert torch.equal(ops.colsum(m.cuda()), ops.colsum(m.cuda()))
    _check_colsum(ops.colsum(m.cuda()), m)
    # a view with ld > cols; the padding must not be read
    buf = torch.full((rows, cols + 6), 1e4, dtype=torch.bfloat16, device="cuda")
    buf[:, :cols] = m.cuda()
    _check_colsum(ops.colsum(buf[:, :cols]), m)


# ----------------------------------------------------------------------------------------------------
# GEMM epilogues on these paths
# ----------------------------------------------------------------------------------------------------
def _gelu_grad64(pre):
    p = pre.double().requires_grad_(True)
    O.gelu(p).backward(torch.ones_like(p))
    return p.grad


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("h", [192, 320, 384])
def test_gemm_gelu_grad_epilogue_at_mlp_backward_shapes(ops, h, block_n):
    """d_pre = (d_mlp_out @ W2) * gelu'(pre) of layer_backward: M = 2 x 128 tokens, N = 4h, K = h, B = W2 [h, 4h]."""
    M, N, K = 256, 4 * h, h
    g = torch.Generator().manual_seed(h + block_n)
    A = bf(torch.randn((M, K), generator=g))
    B = bf(torch.randn((K, N), generator=g) * 0.05)
    aux = bf(torch.randn((M, N), generator=g) * 2)
    out = ops.gemm(A.cuda(), B.cuda(), b_mn_major=True, act=ops.ACT_GELU_GRAD, aux=aux.cuda(), block_n=block_n)
    ref = (A.double() @ B.double()) * _gelu_grad64(aux)
    e = block_err(out, ref)
    assert e < 2e-2, e


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K,with_bias", [(256, 1536, 384, True), (300, 960, 320, False), (200, 1000, 192, True)])
def test_gemm_relu_and_no_bias(ops, M, N, K, with_bias, block_n):
    g = torch.Generator().manual_seed(M + N + K + block_n)
    A, B = bf(torch.randn((M, K), generator=g)), bf(torch.randn((N, K), generator=g) * 0.1)
    bias = bf(torch.randn(N, generator=g)) if with_bias else None
    lin = A.double() @ B.double().t() + (bias.double() if with_bias else 0.0)
    for act, ref in ((ops.ACT_RELU, lin.clamp_min(0)), (ops.ACT_NONE, lin)):
        for dt in (BF16, F32):
            out = ops.gemm(A.cuda(), B.cuda(), bias=bias.cuda() if with_bias else None, act=act, out_dtype=dt,
                           block_n=block_n)
            e = block_err(out, ref)
            assert e < tol(dt), (act, dt, e)
            if act == ops.ACT_RELU:
                assert bool((out >= 0).all())


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(256, 1001, 384), (300, 1001, 320)])
def test_gemm_into_a_row_padded_output_view(ops, M, N, K, block_n):
    """out = buf[:, :N] with ldc > N (the padded logits buffer of _LogitsFn): the padding columns stay untouched."""
    g = torch.Generator().manual_seed(M + K + block_n)
    A, B = bf(torch.randn((M, K), generator=g)), bf(torch.randn((N, K), generator=g) * 0.1)
    ref = A.double() @ B.double().t()
    for dt, ld in ((F32, (N + 3) // 4 * 4), (BF16, (N + 7) // 8 * 8)):
        buf = torch.full((M, ld), float("nan"), dtype=dt, device="cuda")
        out = ops.gemm(A.cuda(), B.cuda(), out_dtype=dt, out=buf[:, :N], block_n=block_n)
        assert out.data_ptr() == buf.data_ptr()
        e = block_err(buf[:, :N], ref)
        assert e < tol(dt), (dt, e)
        assert bool(torch.isnan(buf[:, N:]).all()), dt


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("V,h", [(1001, 320), (1001, 384), (2049, 192)])
def test_gemm_mn_major_a_with_padded_leading_dimension(ops, V, h, block_n):
    """The word-embedding gradient d_w = dl^T @ hidden of _LogitsFn.backward: A = dl [rows, V] as a view of a
    [rows, ceil8(V)] buffer (MN-major, lda > M = V), B = hidden [rows, h] (MN-major), K = rows."""
    rows = 256
    g = torch.Generator().manual_seed(V + h + block_n)
    dl = bf(torch.randn((rows, V), generator=g))
    hid = bf(torch.randn((rows, h), generator=g))
    buf = torch.full((rows, (V + 7) // 8 * 8), 1e3, dtype=torch.bfloat16, device="cuda")
    buf[:, :V] = dl.cuda()
    out = ops.gemm(buf[:, :V], hid.cuda(), a_mn_major=True, b_mn_major=True, block_n=block_n)
    assert out.shape == (V, h)
    e = block_err(out, dl.double().t() @ hid.double())
    assert e < 2e-2, e


# ----------------------------------------------------------------------------------------------------
# GPT2Model training off the 256 grid
# ----------------------------------------------------------------------------------------------------
VOCAB = 1001          # odd: the logits buffer is padded and the logits gradient copied into an aligned buffer


def _gpt2(h, heads, layers, s, *, ckpt=False, max_mem=0, p_emb=0.0, p_attn=0.0, p_out=0.0, seed=5):
    from cogview_b200.model import GPT2Model
    sd = recipes.gpt2_state_dict(num_layers=layers, vocab_size=VOCAB, hidden_size=h, max_sequence_length=s, seed=seed)
    m = GPT2Model(num_layers=layers, vocab_size=VOCAB, hidden_size=h, num_attention_heads=heads,
                  embedding_dropout_prob=p_emb, attention_dropout_prob=p_attn, output_dropout_prob=p_out,
                  max_sequence_length=s, max_memory_length=max_mem, checkpoint_activations=ckpt)
    m.load_state_dict(sd)
    return m.cuda().bfloat16(), sd


def _tokens(b, s, seed):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randint(0, VOCAB, (b, s), generator=g)
    labels = torch.randint(0, VOCAB, (b, s), generator=g)
    return tokens, labels, torch.arange(s).unsqueeze(0).expand(b, -1).contiguous()


def _train_and_compare(m, sd, heads, tokens, labels, pos, *, grad_tol=6e-2, label=""):
    """One training step of m against fp64 autograd of O.gpt2_forward on the bf16-rounded weights (O's self_attention
    / mlp may be monkeypatched by the caller)."""
    from cogview_b200 import mpu
    s = tokens.shape[1]
    logits, *_ = m(tokens.cuda(), pos.cuda(), torch.tril(torch.ones((1, 1, s, s), device="cuda")), None, None, 0)
    losses = mpu.vocab_parallel_cross_entropy(logits.contiguous().float(), labels.cuda())
    losses.mean().backward()
    sdr = {k: v.to(torch.bfloat16).double().requires_grad_(True) for k, v in sd.items()}
    o_logits, _ = O.gpt2_forward(sdr, heads, tokens, pos, torch.tril(torch.ones((1, 1, s, s), dtype=torch.float64)))
    o_losses = O.vocab_parallel_cross_entropy(o_logits, labels)
    o_losses.mean().backward()
    e = row_err(logits, o_logits)
    print("%s logits: worst row error / row scale %.3e" % (label, e))
    assert e < 2e-2, e
    assert (losses.double().cpu() - o_losses.detach()).abs().max().item() < 5e-2
    worst = ("", 0.0, 0.0)
    for n, p in m.named_parameters():
        assert p.grad is not None, n
        ref = sdr[n].grad
        got = p.grad.double().cpu()
        eg = ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()
        er = row_err(got if got.dim() == 2 else got[None], ref if ref.dim() == 2 else ref[None], floor=0.1)
        if er > worst[2]:
            worst = (n, eg, er)
        assert eg < grad_tol and er < grad_tol, (n, eg, er)
    print("%s worst gradient: %s global %.3e, per row %.3e" % ((label,) + worst))
    return logits, losses


@pytest.mark.parametrize("ckpt", [False, True])
@pytest.mark.parametrize("h,heads", [(320, 5), (384, 6)])
def test_model_training_step_off_the_256_grid(h, heads, ckpt):
    """2 layers, vocabulary 1001, b = 2, s = 128: unfused LayerNorm backward, colsum bias gradients, padded logits."""
    m, sd = _gpt2(h, heads, 2, 128, ckpt=ckpt)
    tokens, labels, pos = _tokens(2, 128, seed=h)
    _train_and_compare(m.train(), sd, heads, tokens, labels, pos, label="h=%d ckpt=%s" % (h, ckpt))


def test_model_training_step_at_h3072():
    """(3072, 48), one layer, b = 1, s = 128: the staged LayerNorm forward without a residual (cols > 2560) and the
    fused backward at 3072 columns."""
    m, sd = _gpt2(3072, 48, 1, 128)
    tokens, labels, pos = _tokens(1, 128, seed=3072)
    _train_and_compare(m.train(), sd, 48, tokens, labels, pos, label="h=3072")


# ----------------------------------------------------------------------------------------------------
# dropout off the grid
# ----------------------------------------------------------------------------------------------------
def _dropout_step(ckpt, site_counter):
    from cogview_b200 import mpu
    from cogview_b200.mpu import random as mrandom
    torch.manual_seed(4321)
    mrandom.set_dropout_site_counter(site_counter)
    m, _ = _gpt2(384, 6, 2, 128, ckpt=ckpt, p_emb=P, p_attn=P, p_out=P)
    m.train()
    tokens, labels, pos = _tokens(2, 128, seed=9)
    logits, *_ = m(tokens.cuda(), pos.cuda(), torch.tril(torch.ones((1, 1, 128, 128), device="cuda")), None, None, 0)
    loss = mpu.vocab_parallel_cross_entropy(logits.contiguous().float(), labels.cuda()).mean()
    loss.backward()
    return loss.item(), {n: p.grad.float().clone() for n, p in m.named_parameters()}


@pytest.mark.parametrize("p", [0.0, P])
def test_embedding_bwd_with_repeated_ids_is_deterministic(ops, p):
    """A small vocabulary repeats tokens many times per batch (and every position repeats once per sequence): the
    table gradients must be the same bits on every run, and match the fp64 scatter-add of dx (through the dropout
    mask of the embedding site)."""
    rows, h, V, S = 256, 320, VOCAB, 128
    g = torch.Generator().manual_seed(21)
    ids = torch.randint(0, 20, (rows,), generator=g)
    pos = torch.arange(rows) % S
    dx = torch.randn((rows, h), generator=g)
    drop = (p, 99, 4) if p > 0 else None
    outs = []
    for _ in range(2):
        dwte = torch.zeros((V, h), dtype=torch.bfloat16, device="cuda")
        dwpe = torch.zeros((S, h), dtype=torch.bfloat16, device="cuda")
        ops.embed_bwd(ids.cuda(), pos.cuda(), dx.cuda(), dwte, dwpe, dropout=drop)
        outs.append((dwte, dwpe))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    if p == 0:
        # every position occurs exactly twice: bf16(bf16(dx[r]) + bf16(dx[r + S])), as two bf16 atomic adds give
        two = (bf(dx[:S]).float() + bf(dx[S:]).float()).to(torch.bfloat16)
        assert torch.equal(outs[0][1].cpu(), two)
    d = dx.double()
    if p > 0:
        d = d * ops.dropout_mask(rows * h, p, 99, 4).view(rows, h).cpu().double() / (1 - p)
    r1 = torch.zeros((V, h), dtype=torch.float64).index_add_(0, ids, d)
    r2 = torch.zeros((S, h), dtype=torch.float64).index_add_(0, pos, d)
    assert bool((outs[0][0][20:] == 0).all())
    assert row_err(outs[0][0][:20], r1[:20]) < 3e-2 and row_err(outs[0][1], r2) < 2e-2


def test_training_with_dropout_at_h384_is_reproducible_and_checkpoint_safe():
    l0, g0 = _dropout_step(False, 100)
    l1, g1 = _dropout_step(False, 100)
    l2, g2 = _dropout_step(True, 100)        # activation checkpointing regenerates the same masks
    l3, _ = _dropout_step(False, 500)        # other sites, other masks
    assert l0 == l1 and [n for n in g0 if not torch.equal(g0[n], g1[n])] == []
    assert abs(l0 - l2) < 1e-6 and max((g0[n] - g2[n]).abs().max().item() for n in g0) < 1e-6
    assert l3 != l0
    assert 3.0 < l0 < 20.0 and all(torch.isfinite(v).all() for v in g0.values())


def test_output_dropout_at_h384_matches_oracle(monkeypatch):
    """output_dropout_prob = 0.1, the other dropouts 0: the oracle applies each layer's keep masks of the attention
    output ('out', second site of the layer) and the MLP output ('mlp', third site), regenerated with
    ops.dropout_mask from the layer's (seed, site), before third_layernorm / fourth_layernorm."""
    from cogview_b200 import ops
    from cogview_b200.mpu import random as mrandom
    h, heads, b, s, c0 = 384, 6, 2, 128, 2000
    torch.manual_seed(4321)
    mrandom.set_dropout_site_counter(c0)
    m, sd = _gpt2(h, heads, 2, s, p_out=P)
    tokens, labels, pos = _tokens(b, s, seed=17)
    seed = torch.initial_seed()

    def keep(site):
        return ops.dropout_mask(b * s * h, P, seed, site).view(b, s, h).cpu().double() / (1 - P)
    keep_out = [keep(c0 + 3 * li + 2) for li in range(2)]
    keep_mlp = [keep(c0 + 3 * li + 3) for li in range(2)]
    orig_sa, orig_mlp = O.self_attention, O.mlp

    def layer_of(pre):               # 'transformer.layers.<i>.attention.' / 'transformer.layers.<i>.mlp.'
        return int(pre.split('.')[2])

    def self_attention(sd_, pre, x, *a, **k):
        return orig_sa(sd_, pre, x, *a, **k) * keep_out[layer_of(pre)]

    def mlp(sd_, pre, x):
        return orig_mlp(sd_, pre, x) * keep_mlp[layer_of(pre)]
    monkeypatch.setattr(O, "self_attention", self_attention)
    monkeypatch.setattr(O, "mlp", mlp)
    _train_and_compare(m.train(), sd, heads, tokens, labels, pos, label="h=384 output dropout")
    monkeypatch.undo()


# ----------------------------------------------------------------------------------------------------
# decode off the grid
# ----------------------------------------------------------------------------------------------------
def test_kv_decode_at_h320_matches_full_prefix_forward(monkeypatch):
    """Prefill 64 tokens, then 16 single-token steps through the K|V-cache decode graph; each step's logits against a
    no-memory forward over the whole prefix with the same weights."""
    monkeypatch.setenv("COGVIEW_B200_CUDA_GRAPH", "1")
    h, heads, b, n0, n = 320, 5, 2, 64, 16
    m, _ = _gpt2(h, heads, 2, 128, max_mem=128)
    m.transformer.mems_mode = "kv"
    m.eval()
    ref_model, _ = _gpt2(h, heads, 2, 128)
    ref_model.eval()
    tokens, _, pos = _tokens(b, n0 + n, seed=320)
    tokens, pos = tokens.cuda(), pos.cuda()
    worst = 0.0
    with torch.no_grad():
        lg, *mems = m(tokens[:, :n0], pos[:, :n0], torch.tril(torch.ones((1, 1, n0, n0), device="cuda")), None, None, 0)
        for t in range(n0, n0 + n):
            lg, *mems = m(tokens[:, t:t + 1], pos[:, t:t + 1], 0, None, None, 0, *mems)
            assert mems[0].size(1) == t + 1
            full, *_ = ref_model(tokens[:, :t + 1], pos[:, :t + 1],
                                 torch.tril(torch.ones((1, 1, t + 1, t + 1), device="cuda")), None, None, 0)
            e = row_err(lg[:, -1], full[:, -1])
            worst = max(worst, e)
            assert e < 2e-2, (t, e)
    runner = m.transformer._kv.runner
    print("h=320 decode: worst step logits error / row scale %.3e, graph replays %d" % (worst, runner.replays))
    assert runner.replays == n


def _ln_small_m_ref(res, go, gp, bp, gq, bq):
    y = res.double() + O.layernorm_absmax(go.double(), gp.double(), bp.double())
    return y, O.layernorm_absmax(y, gq.double(), bq.double())


@pytest.mark.parametrize("M", [1, 3, 9, 16])
@pytest.mark.parametrize("K", [320, 384, 3072, 5120])
def test_ln_pair_small_m_off_the_grid(ops, M, K):
    g = torch.Generator().manual_seed(M * K + 1)
    res = torch.randn((M, K), generator=g) * (10.0 ** (torch.rand((M, 1), generator=g) * 2 - 1))
    go = bf(torch.randn((M, K), generator=g) * 5)
    gp, bp = bf(1 + 0.1 * torch.randn(K, generator=g)), bf(0.1 * torch.randn(K, generator=g))
    gq, bq = bf(1 + 0.1 * torch.randn(K, generator=g)), bf(0.1 * torch.randn(K, generator=g))
    y_ref, xn_ref = _ln_small_m_ref(res, go, gp, bp, gq, bq)
    y, xn = ops.ln_pair_small_m(res.cuda(), go.cuda(), ops.absmax(go.cuda()), (gp.cuda(), bp.cuda()),
                                (gq.cuda(), bq.cuda()), O.LN_EPS)
    assert row_err(y, y_ref) < 1e-4 and row_err(xn, xn_ref) < 2e-2
    _, xn0 = ops.ln_pair_small_m(res.cuda(), None, None, None, (gq.cuda(), bq.cuda()), O.LN_EPS, want_res_out=False)
    assert row_err(xn0, O.layernorm_absmax(res.double(), gq.double(), bq.double())) < 2e-2


@pytest.mark.parametrize("M", [1, 3, 9, 16])
@pytest.mark.parametrize("K", [320, 384])
def test_linear_small_m_off_the_grid(ops, M, K):
    """The decode linears at h = 320 / 384: QKV (N = 3K), MLP (N = 4K, GELU) and the logits (N = 1001, fp32 rows of
    odd length)."""
    for N, act in ((3 * K, ops.ACT_NONE), (4 * K, ops.ACT_GELU), (VOCAB, ops.ACT_NONE)):
        g = torch.Generator().manual_seed(M + N + K)
        x, w = bf(torch.randn((M, K), generator=g)), bf(torch.randn((N, K), generator=g) * 0.05)
        bias = bf(torch.randn(N, generator=g))
        ref = x.double() @ w.double().t() + bias.double()
        if act == ops.ACT_GELU:
            ref = O.gelu(ref)
        am = torch.zeros(1, device="cuda")
        out = ops.linear_small_m(x.cuda(), w.cuda(), bias.cuda(), act=act, absmax=am)
        assert row_err(out, ref) < 2e-2, (N, act)
        assert am.item() == out.float().abs().max().item()
        out32 = ops.linear_small_m(x.cuda(), w.cuda(), bias.cuda(), act=act, out_dtype=torch.float32)
        assert row_err(out32, ref) < 1e-4, (N, act)


# ----------------------------------------------------------------------------------------------------
# cross entropy at V % 4 != 0
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1001, 1002, 1003])
@pytest.mark.parametrize("layout", ["contiguous", "sliced"])
def test_vocab_parallel_cross_entropy_odd_vocab(V, layout):
    """mpu.vocab_parallel_cross_entropy on fp32 logits [b, s, V] with V % 4 != 0: contiguous (rows not 16-byte
    aligned), or a [:, :, :V] slice of a [b, s, V + 1] tensor (aligned rows only for V = 1003)."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import mpu
    b, s = 2, 64
    g = torch.Generator().manual_seed(V)
    full = torch.randn((b, s, V + 1), generator=g) * 4
    target = torch.randint(0, V, (b, s), generator=g)
    gl = torch.rand((b, s), generator=g)
    src = (full[..., :V].contiguous() if layout == "contiguous" else full).cuda().requires_grad_(True)
    logits = src[..., :V]
    loss = mpu.vocab_parallel_cross_entropy(logits, target.cuda())
    loss.backward(gl.cuda())
    lr = full[..., :V].double().requires_grad_(True)
    ref = O.vocab_parallel_cross_entropy(lr, target)
    ref.backward(gl.double())
    assert loss.shape == (b, s)
    assert (loss.double().cpu() - ref.detach()).abs().max().item() < 1e-4
    e = row_err(src.grad[..., :V], lr.grad)
    assert e < 4e-3, e
