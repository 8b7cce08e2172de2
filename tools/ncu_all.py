"""One profiled pass over every kernel family of the path, for `ncu --set full`.

    ncu --set full --clock-control none --import-source on --profile-from-start off -o gpurun_out/r02_<group> \
        python tools/ncu_all.py <group>

groups:  train   GEMM (qkv shape), attention fwd / bwd (dense with dropout, sparse), LayerNorm fwd / bwd, embedding,
                 cross-entropy fwd / bwd, colsum, multi-tensor sum-of-squares + AdamW (a 4-layer model's parameters)
         decode  small-M linear (qkv shape, M = 4 and 16), Sandwich-LN glue, cached attention, gathered (sparse) attention,
                 sampling epilogue
         vqvae   conv / transposed conv (wgmma implicit GEMM), im2col, split + distance GEMM + arg-min + lookup, 1x1-to-RGB
Each kernel runs twice untimed first; inputs are larger than L2 or the L2 is flushed before the profiled launch."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from cogview_b200 import ops  # noqa: E402

flush_buf = None


def flush():
    global flush_buf
    if flush_buf is None:
        flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    flush_buf.zero_()


def profiled(fns):
    for _ in range(2):
        for f in fns:
            f()
    torch.cuda.synchronize()
    for f in fns:
        flush()
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        f()
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()


def bf(t):
    return t.to(torch.bfloat16)


def train():
    g = torch.Generator(device="cuda").manual_seed(0)
    b, s, heads = 4, 1088, 40
    h = heads * 64
    M = b * s
    x = bf(torch.randn((M, h), generator=g, device="cuda"))
    wqkv = bf(torch.randn((3 * h, h), generator=g, device="cuda") * 0.02)
    bias = bf(torch.randn(3 * h, generator=g, device="cuda"))
    qkv = bf(torch.randn((b, s, 3 * h), generator=g, device="cuda") * 0.5)
    d_out = bf(torch.randn((b, s, h), generator=g, device="cuda"))
    q, k, v = qkv[..., :h], qkv[..., h:2 * h], qkv[..., 2 * h:]
    out, lse, mask = ops.attn_fwd(q, k, v, heads, want_lse=True, dropout=(0.1, 11, 3))
    import random
    random.seed(0)
    s_sp = 1024
    piv = torch.stack([torch.tensor(sorted(random.sample(range(s_sp), 768)), dtype=torch.long) for _ in range(b)]).cuda()
    qs, ks, vs = q[:, :s_sp], k[:, :s_sp], v[:, :s_sp]
    xf = torch.randn((M, h), generator=g, device="cuda")
    gamma = torch.ones(h, dtype=torch.bfloat16, device="cuda")
    beta = torch.zeros(h, dtype=torch.bfloat16, device="cuda")
    am = torch.full((1,), 5.0, device="cuda")
    amo = torch.zeros(1, device="cuda")
    _, mean, rstd = ops.layernorm_absmax_fwd(xf, am, gamma, beta, 1e-5, save_stats=True)
    V = 58240
    logits = torch.randn((M, V), generator=g, device="cuda")
    tgt = torch.randint(0, V, (M,), generator=g, device="cuda")
    ce = ops.cross_entropy_fwd(logits, tgt)
    from bench import build_model
    from cogview_b200.model import gpt2_get_params_for_weight_decay_optimization
    from cogview_b200.optim import FusedAdamW
    small = build_model(dict(num_layers=4, vocab_size=58240, hidden_size=2560, num_attention_heads=40,
                             max_sequence_length=1089), 0, "cuda").train()
    opt = FusedAdamW(gpt2_get_params_for_weight_decay_optimization(small), lr=1e-4, weight_decay=0.01, max_grad_norm=1.0)
    for p in small.parameters():
        p.grad = torch.randn_like(p) * 0.01
    ids = torch.randint(0, V, (b, s), generator=g, device="cuda")
    pos = torch.arange(s, device="cuda").unsqueeze(0).expand(b, -1).contiguous()
    wte = bf(torch.randn((V, h), generator=g, device="cuda") * 0.02)
    wpe = bf(torch.randn((1089, h), generator=g, device="cuda") * 0.02)
    profiled([
        lambda: ops.gemm(x, wqkv, bias=bias),
        lambda: ops.attn_fwd(q, k, v, heads, want_lse=True, dropout=(0.1, 11, 3)),
        lambda: ops.attn_bwd(q, k, v, out, d_out, lse, heads, dropout_p=0.1, drop_mask=mask),
        lambda: ops.attn_sparse_fwd(qs, ks, vs, heads, piv, 128, 6, want_lse=True),
        lambda: ops.layernorm_absmax_fwd(xf, am, gamma, beta, 1e-5, save_stats=True),
        lambda: ops.layernorm_absmax_fwd(x, am, gamma, beta, 1e-5, residual=xf, out_dtype=torch.float32, absmax_out=amo,
                                         save_stats=True),
        lambda: ops.layernorm_absmax_bwd(xf, x, mean, rstd, gamma, dres=xf, dx_dtype=torch.float32),
        lambda: ops.layernorm_absmax_bwd(x, xf, mean, rstd, gamma, dx_dtype=torch.bfloat16, want_dxsum=True),
        lambda: ops.embed_fwd(ids, pos, wte, wpe, amo),
        lambda: ops.cross_entropy_fwd(logits, tgt),
        lambda: ops.cross_entropy_bwd(logits, tgt, ce[1], ce[2], torch.full((M,), 1.0 / M, device="cuda")),
        lambda: ops.colsum(x),
        lambda: opt.step(),
    ])


def decode():
    g = torch.Generator(device="cuda").manual_seed(0)
    h, heads, M = 2560, 40, 4
    w = bf(torch.randn((3 * h, h), generator=g, device="cuda") * 0.02)
    bias = bf(torch.randn(3 * h, generator=g, device="cuda"))
    x4 = bf(torch.randn((4, h), generator=g, device="cuda"))
    x16 = bf(torch.randn((16, h), generator=g, device="cuda"))
    res = torch.randn((M, h), generator=g, device="cuda")
    go = bf(torch.randn((M, h), generator=g, device="cuda") * 3)
    am = go.float().abs().max().reshape(1)
    gam = torch.ones(h, dtype=torch.bfloat16, device="cuda")
    bet = torch.zeros(h, dtype=torch.bfloat16, device="cuda")
    t = 1000
    cache = bf(torch.randn((M, 1089, 2 * h), generator=g, device="cuda") * 0.5)
    qkv = bf(torch.randn((M, 3 * h), generator=g, device="cuda") * 0.5)
    idx = torch.stack([torch.randperm(t, generator=torch.Generator().manual_seed(i))[:768 + 128].sort().values for i in range(M)]).cuda()
    logits = torch.randn((M, 58240), generator=g, device="cuda")
    next_ids = torch.zeros((M, 1), dtype=torch.int64, device="cuda")
    fns = [
        lambda: ops.linear_small_m(x4, w, bias),
        lambda: ops.linear_small_m(x16, w, bias),
        lambda: ops.ln_pair_small_m(res, go, am, (gam, bet), (gam, bet), 1e-5),
        lambda: ops.attn_decode(qkv, cache, heads, cur_len=t, nsplit=8),
        lambda: ops.attn_gather(qkv[:, :h].reshape(M, 1, h), cache[:, :t], idx, heads),
        lambda: ops.sample_topk(logits, 1.0, 200, [(0, 8192)], seed=1, next_ids=next_ids),
    ]
    profiled(fns)


def vqvae():
    from cogview_b200 import recipes
    from cogview_b200 import vqvae as vq
    model = vq.new_model()
    model.load_state_dict(recipes.vqvae_state_dict(seed=0))
    model = model.cuda().eval()
    img = torch.randn((16, 3, 256, 256), device="cuda")

    def roundtrip():
        codes = vq.img2code(model, img)
        vq.code2img(model, codes.view(16, 32, 32))
    profiled([roundtrip])


if __name__ == "__main__":
    {"train": train, "decode": decode, "vqvae": vqvae}[sys.argv[1] if len(sys.argv) > 1 else "train"]()
