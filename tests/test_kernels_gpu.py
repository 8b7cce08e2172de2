"""GPU parity tests of the individual C-ABI kernels against the CPU oracle (oracle/cogview_oracle.py) on
seeded inputs.  Tolerances: bf16 outputs are compared at 2e-2 of the tensor scale (bf16 has 8 mantissa
bits; inputs are rounded to bf16 before the oracle sees them, so only accumulation order and the final
rounding differ); fp32 outputs at 1e-4."""
import pytest
import torch

from oracle import cogview_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


def rel_err(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def bf(x):
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(256, 768, 256, 0, 0), (200, 328, 136, 0, 0), (256, 256, 1024, 0, 1),
                                             (256, 1024, 256, 1, 1), (4352, 2560, 2560, 0, 0)])
def test_gemm_matches_fp32_matmul(ops, M, N, K, a_mn, b_mn):
    g = torch.Generator().manual_seed(M + N + K)
    A = bf(torch.randn((K, M) if a_mn else (M, K), generator=g))
    B = bf(torch.randn((K, N) if b_mn else (N, K), generator=g))
    bias = bf(torch.randn(N, generator=g))
    ref = (A.float().t() if a_mn else A.float()) @ (B.float() if b_mn else B.float().t()) + bias.float()
    out = ops.gemm(A.cuda(), B.cuda(), a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), bias=bias.cuda())
    assert rel_err(out, ref) < 1e-2
    out32 = ops.gemm(A.cuda(), B.cuda(), a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), bias=bias.cuda(),
                     out_dtype=torch.float32)
    assert rel_err(out32, ref) < 1e-4


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(200, 328, 136, 0, 0), (384, 640, 192, 0, 1), (320, 1000, 256, 1, 1),
                                             (4352, 2560, 512, 0, 0), (4352, 2560, 512, 0, 1), (2560, 2560, 1088, 1, 1),
                                             (19000, 512, 128, 0, 0)])
def test_gemm_tail_wave_split(ops, M, N, K, a_mn, b_mn):
    """256-wide tile schedule whose last partial wave is issued as half-width tiles (gemm.cu tile_coord): small
    shapes (every tile split, ragged N with a fully out-of-range half), the 4B layer shapes (2 full waves + 44 split
    tiles) and a shape with many full waves before the split tail; bf16 and fp32 outputs, all operand layouts."""
    g = torch.Generator().manual_seed(M + N + K + a_mn)
    A = bf(torch.randn((K, M) if a_mn else (M, K), generator=g))
    B = bf(torch.randn((K, N) if b_mn else (N, K), generator=g))
    bias = bf(torch.randn(N, generator=g))
    ref = (A.float().t() if a_mn else A.float()) @ (B.float() if b_mn else B.float().t()) + bias.float()
    for dt, tol in ((torch.bfloat16, 1e-2), (torch.float32, 1e-4)):
        out = ops.gemm(A.cuda(), B.cuda(), a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), bias=bias.cuda(),
                       out_dtype=dt, block_n=256)
        diff = (out.float().cpu() - ref).abs()
        assert diff.max().item() / ref.abs().max().item() < tol
        # every 128 x 128 block individually (a dropped half tile in a corner must not hide behind a global max)
        blk = torch.nn.functional.max_pool2d(diff[None, None], 128, ceil_mode=True)[0, 0]
        assert (blk < tol * ref.abs().max()).all()


def test_gemm_gelu_preact_absmax(ops):
    g = torch.Generator().manual_seed(3)
    A, B, bias = bf(torch.randn((384, 256), generator=g)), bf(torch.randn((1024, 256), generator=g) * 0.1), bf(
        torch.randn(1024, generator=g))
    pre_ref = A.float() @ B.float().t() + bias.float()
    act_ref = O.gelu(pre_ref)
    am = torch.zeros(1, device="cuda")
    out, pre = ops.gemm(A.cuda(), B.cuda(), bias=bias.cuda(), act=ops.ACT_GELU, absmax=am, want_preact=True)
    assert rel_err(pre, pre_ref) < 1e-2 and rel_err(out, act_ref) < 1e-2
    assert am.item() == out.float().abs().max().item()


@pytest.mark.parametrize("rows,cols", [(256, 256), (100, 2560)])
def test_layernorm_absmax_fwd_bwd(ops, rows, cols):
    g = torch.Generator().manual_seed(rows)
    x = torch.randn((rows, cols), generator=g) * 3.0
    x[0, 0] = 40.0                                    # an outlier sets the global scale
    gamma, beta = bf(1 + 0.1 * torch.randn(cols, generator=g)), bf(0.1 * torch.randn(cols, generator=g))
    res = torch.randn((rows, cols), generator=g)
    # (1) fp32 in -> bf16 out (input / post-attention / final LN)
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.float().requires_grad_(True), beta.float().requires_grad_(True)
    y_ref = O.layernorm_absmax(xr, gr, br)
    am = ops.absmax(x.cuda())
    assert am.item() == x.abs().max().item()
    y, mean, rstd = ops.layernorm_absmax_fwd(x.cuda(), am, gamma.cuda(), beta.cuda(), 1e-5, save_stats=True)
    assert rel_err(y, y_ref.detach()) < 1e-2
    dy = bf(torch.randn((rows, cols), generator=g))
    dres = torch.randn((rows, cols), generator=g)
    y_ref.backward(dy.float())
    dx, dg, db = ops.layernorm_absmax_bwd(x.cuda(), dy.cuda(), mean, rstd, gamma.cuda(), dres=dres.cuda())
    assert rel_err(dx, xr.grad + dres) < 1e-4
    assert rel_err(dg, gr.grad) < 1e-2 and rel_err(db, br.grad) < 1e-2
    # (2) bf16 in -> fp32 out with residual (third / fourth LN), abs-max of the result
    xb = bf(x)
    xr2 = xb.float().requires_grad_(True)
    y2_ref = res + O.layernorm_absmax(xr2, gamma.float(), beta.float())
    am2, amo = ops.absmax(xb.cuda()), torch.zeros(1, device="cuda")
    y2, mean2, rstd2 = ops.layernorm_absmax_fwd(xb.cuda(), am2, gamma.cuda(), beta.cuda(), 1e-5, residual=res.cuda(),
                                                out_dtype=torch.float32, absmax_out=amo, save_stats=True)
    assert rel_err(y2, y2_ref.detach()) < 1e-4
    assert abs(amo.item() - y2.abs().max().item()) == 0.0
    dy2 = torch.randn((rows, cols), generator=g)
    y2_ref.backward(dy2)
    dx2, _, _ = ops.layernorm_absmax_bwd(xb.cuda(), dy2.cuda(), mean2, rstd2, gamma.cuda(), dx_dtype=torch.bfloat16)
    assert rel_err(dx2, xr2.grad) < 1e-2
    # (3) the fused kernel's extra output: column sums of dx (bias gradient of the producing linear layer)
    dx3, dg3, db3, dxsum = ops.layernorm_absmax_bwd(xb.cuda(), dy2.cuda(), mean2, rstd2, gamma.cuda(),
                                                    dx_dtype=torch.bfloat16, want_dxsum=True)
    assert torch.equal(dx3, dx2)
    assert rel_err(dxsum, dx2.float().sum(0)) < 1e-2


def test_embedding_fwd_bwd(ops):
    g = torch.Generator().manual_seed(5)
    V, P, h, rows = 1000, 128, 256, 300
    wte, wpe = bf(torch.randn((V, h), generator=g)), bf(torch.randn((P, h), generator=g))
    ids, pos = torch.randint(0, V, (rows,), generator=g), torch.randint(0, P, (rows,), generator=g)
    am = torch.zeros(1, device="cuda")
    out = ops.embed_fwd(ids.cuda(), pos.cuda(), wte.cuda(), wpe.cuda(), am)
    ref = wte.float()[ids] + wpe.float()[pos]
    assert rel_err(out, ref) < 1e-6 and am.item() == ref.abs().max().item()
    dx = torch.randn((rows, h), generator=g)
    dwte, dwpe = torch.zeros((V, h), dtype=torch.bfloat16, device="cuda"), torch.zeros((P, h), dtype=torch.bfloat16,
                                                                                       device="cuda")
    ops.embed_bwd(ids.cuda(), pos.cuda(), dx.cuda(), dwte, dwpe)
    r1 = torch.zeros((V, h)).index_add_(0, ids, dx)
    r2 = torch.zeros((P, h)).index_add_(0, pos, dx)
    assert rel_err(dwte, r1) < 2e-2 and rel_err(dwpe, r2) < 3e-2


@pytest.mark.parametrize("rows,V", [(64, 58240), (33, 1003)])
def test_cross_entropy_fwd_bwd(ops, rows, V):
    g = torch.Generator().manual_seed(V)
    ld = (V + 3) // 4 * 4
    logits = torch.randn((rows, ld), generator=g) * 4
    target = torch.randint(0, V, (rows,), generator=g)
    lr = logits[:, :V].clone().requires_grad_(True)
    ref = O.vocab_parallel_cross_entropy(lr, target)
    lg = logits.cuda()[:, :V]
    loss, rmax, rsum = ops.cross_entropy_fwd(lg, target.cuda())
    assert (loss.cpu() - ref.detach()).abs().max().item() < 1e-4
    gl = torch.rand(rows, generator=g)
    ref.backward(gl)
    dl = ops.cross_entropy_bwd(lg, target.cuda(), rmax, rsum, gl.cuda())
    assert (dl.float().cpu() - lr.grad).abs().max().item() < 4e-3 * lr.grad.abs().max().item() + 1e-6


def test_gelu_bwd_and_colsum(ops):
    g = torch.Generator().manual_seed(9)
    pre, dact = bf(torch.randn((128, 1024), generator=g) * 2), bf(torch.randn((128, 1024), generator=g))
    pr = pre.float().requires_grad_(True)
    O.gelu(pr).backward(dact.float())
    assert rel_err(ops.gelu_bwd(pre.cuda(), dact.cuda()), pr.grad) < 1e-2
    assert rel_err(ops.colsum(dact.cuda()), dact.float().sum(0)) < 1e-2


def test_fused_adamw_matches_torch_adamw_on_fp32_masters(ops):
    """Multi-tensor AdamW + global-norm clipping over two parameter groups (weight decay / no weight decay,
    gpt2_get_params_for_weight_decay_optimization) against torch.optim.AdamW on fp32 copies."""
    from cogview_b200.optim import FusedAdamW
    g = torch.Generator().manual_seed(11)
    shapes = [(300, 257), (2560,), (7,), (1024, 64)]
    w0 = [torch.randn(sh, generator=g) for sh in shapes]
    ps = [torch.nn.Parameter(bf(w).cuda()) for w in w0]
    refs = [torch.nn.Parameter(bf(w).float()) for w in w0]
    opt = FusedAdamW([{'params': [ps[0], ps[3]], 'weight_decay': 0.01}, {'params': [ps[1], ps[2]], 'weight_decay': 0.0}],
                     lr=1e-2, betas=(0.9, 0.95), eps=1e-8, max_grad_norm=1.0)
    ropt = torch.optim.AdamW([{'params': [refs[0], refs[3]], 'weight_decay': 0.01},
                              {'params': [refs[1], refs[2]], 'weight_decay': 0.0}], lr=1e-2, betas=(0.9, 0.95), eps=1e-8)
    for it in range(3):
        for p, r, sh in zip(ps, refs, shapes):
            gr = bf(torch.randn(sh, generator=g))
            p.grad = gr.cuda()
            r.grad = gr.float().clone()
        gn = torch.nn.utils.clip_grad_norm_(refs, 1.0)
        opt.step()
        ropt.step()
        assert abs(opt.last_grad_norm.item() - gn.item()) < 1e-3 * gn.item()
    for p, r in zip(ps, refs):
        master = opt.state[p]['master'].cpu()
        assert (master - r.detach()).abs().max().item() < 1e-5
        assert torch.equal(p.detach().cpu(), bf(master))


@pytest.mark.parametrize("M,N,K,act", [(4, 7680, 2560, 0), (4, 2560, 10240, 0), (2, 1024, 256, 1), (1, 58240, 256, 0),
                                       (8, 2560, 2560, 0), (13, 520, 264, 0), (16, 2560, 2560, 0), (9, 10240, 2560, 1)])
def test_linear_small_m(ops, M, N, K, act):
    g = torch.Generator().manual_seed(M + N)
    x, w, bias = bf(torch.randn((M, K), generator=g)), bf(torch.randn((N, K), generator=g) * 0.05), bf(
        torch.randn(N, generator=g))
    ref = x.float() @ w.float().t() + bias.float()
    if act:
        ref = O.gelu(ref)
    am = torch.zeros(1, device="cuda")
    out = ops.linear_small_m(x.cuda(), w.cuda(), bias.cuda(), act=act, absmax=am)
    assert rel_err(out, ref) < 1e-2
    assert am.item() == out.float().abs().max().item()
    out32 = ops.linear_small_m(x.cuda(), w.cuda(), bias.cuda(), act=act, out_dtype=torch.float32)
    assert rel_err(out32, ref) < 1e-5


@pytest.mark.parametrize("M,K", [(4, 2560), (2, 256), (1, 2560), (7, 512), (16, 2560)])
def test_ln_pair_small_m(ops, M, K):
    g = torch.Generator().manual_seed(M * K)
    res = torch.randn((M, K), generator=g)
    go = bf(torch.randn((M, K), generator=g) * 5)
    gp, bp = bf(1 + 0.1 * torch.randn(K, generator=g)), bf(0.1 * torch.randn(K, generator=g))
    gq, bq = bf(1 + 0.1 * torch.randn(K, generator=g)), bf(0.1 * torch.randn(K, generator=g))
    y_ref = res + O.layernorm_absmax(go.float(), gp.float(), bp.float())
    xn_ref = O.layernorm_absmax(y_ref, gq.float(), bq.float())
    am = ops.absmax(go.cuda())
    y, xn = ops.ln_pair_small_m(res.cuda(), go.cuda(), am, (gp.cuda(), bp.cuda()), (gq.cuda(), bq.cuda()), 1e-5)
    assert rel_err(y, y_ref) < 1e-5 and rel_err(xn, xn_ref) < 1e-2
    _, xn0 = ops.ln_pair_small_m(res.cuda(), None, None, None, (gq.cuda(), bq.cuda()), 1e-5, want_res_out=False)
    assert rel_err(xn0, O.layernorm_absmax(res, gq.float(), bq.float())) < 1e-2


def test_attn_gather_matches_sparse_attention_inference(ops, golden_dir):
    """cv_attn_gather vs the oracle's sparse_attention_inference and the reference's golden output."""
    import os
    import numpy as np
    g = np.load(os.path.join(golden_dir, "attention.npz"))
    b, nh, s, hn, w, times, n_piv, sq = [int(x) for x in g["dims"]]
    gen = torch.Generator().manual_seed(int(g["seed"]))
    q, k, v = (torch.randn((b, nh, s, hn), generator=gen) for _ in range(3))
    pivot_idx = torch.from_numpy(g["pivot_idx"])
    pw = torch.cat((pivot_idx, torch.arange(s - times * w, s).expand(b, -1)), dim=-1)
    qb, kb, vb = bf(q), bf(k), bf(v)
    ref = O.sparse_attention_inference(qb.float()[:, :, -sq:], kb.float(), vb.float(), pw)
    from cogview_b200.mpu.sparse_transformer import sparse_attention_inference
    out = sparse_attention_inference(qb[:, :, -sq:].cuda(), kb.cuda(), vb.cuda(), pw.cuda())
    assert rel_err(out, ref) < 1e-2
    assert np.abs(out.float().cpu().numpy() - g["sparse_infer"]).max() < 2e-2 * np.abs(g["sparse_infer"]).max()


@pytest.mark.parametrize("b,heads,t,nsplit", [(2, 3, 0, 1), (2, 3, 0, 4), (1, 2, 5, 16), (3, 2, 63, 1), (2, 4, 64, 3),
                                              (2, 2, 257, 8), (1, 40, 1087, 8)])
def test_attn_decode_kernel_matches_softmax_attention(ops, b, heads, t, nsplit):
    """One query per sequence over t cached keys + the appended one (mpu/sparse_transformer.py:652-673 with the
    mems of :617-634), every key-range split count including splits that receive no key."""
    g = torch.Generator().manual_seed(t + nsplit)
    h, max_len = heads * 64, 1089
    qkv = bf(torch.randn((b, 3 * h), generator=g))
    cache = bf(torch.randn((b, max_len, 2 * h), generator=g))
    cache_dev = cache.cuda()
    out = ops.attn_decode(qkv.cuda(), cache_dev, heads, cur_len=t, nsplit=nsplit)
    # the kernel appended the new K | V at position t
    assert torch.equal(cache_dev[:, t].cpu(), qkv[:, h:])
    assert torch.equal(cache_dev[:, :t].cpu(), cache[:, :t])
    q = qkv[:, :h].float().view(b, heads, 1, 64)
    kv = torch.cat((cache[:, :t].float(), qkv[:, None, h:].float()), dim=1)              # [b, t+1, 2h]
    k = kv[..., :h].view(b, t + 1, heads, 64).permute(0, 2, 1, 3)
    v = kv[..., h:].view(b, t + 1, heads, 64).permute(0, 2, 1, 3)
    ref = torch.matmul(torch.softmax(torch.matmul(q / 8.0, k.transpose(-1, -2)), -1), v).reshape(b, h)
    assert rel_err(out, ref) < 1e-2
