"""ShardedFusedAdamW (ZeRO stage 1, cogview_b200/optim.py) on the GPU against FusedAdamW: at world size 1 through
pretrain.train_step, as "virtual shards" (every rank's step of an N-rank layout run in one process on the same
averaged gradients, the all-reduce and the all-gather done by hand), the gradient views across zero_grad and
backward, a sharded -> consolidated -> FusedAdamW checkpoint, and two ranks under NCCL when two GPUs are visible.

cv_sumsq_bf16_multi adds its per-block partial sums with atomicAdd, so the gradient norm of two runs on the same
gradients - FusedAdamW against itself included - may differ in its last bits.  Where a comparison is bit for bit the
clip coefficient is exactly 1 (no clipping, or a max_grad_norm the norm stays below); with a binding clip the
results agree within the bound stated at _close_after_clip."""
import os
import socket

import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu

VOCAB = 8192 + 1024


def _model(h, ckpt=False, seed=1234):
    from cogview_b200.model import GPT2Model, gpt2_get_params_for_weight_decay_optimization
    cfg = dict(num_layers=2, vocab_size=VOCAB, hidden_size=h, num_attention_heads=h // 64, max_sequence_length=128)
    m = GPT2Model(num_layers=2, vocab_size=VOCAB, hidden_size=h, num_attention_heads=h // 64,
                  embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                  max_sequence_length=128, max_memory_length=0, checkpoint_activations=ckpt)
    m.load_state_dict(recipes.gpt2_state_dict(seed=seed, **cfg))
    m = m.cuda().bfloat16().train()
    groups = gpt2_get_params_for_weight_decay_optimization(m)
    groups[0]['lr'] = 2e-3                     # the two groups differ in lr as well as in weight decay
    return m, groups


def _batch(b=2, seed=3):
    from cogview_b200.generation.sampling import get_masks_and_position_ids
    tf = recipes.text_image_tokens(b, 32, 33, seed=seed, vocab_size=VOCAB).cuda()
    tokens, labels = tf[:, :-1].contiguous(), tf[:, 1:].contiguous()
    mask, loss_mask, pos = get_masks_and_position_ids(tokens)
    return (tokens, labels, loss_mask, mask, pos)


def _opt(cls, groups, max_grad_norm, **kw):
    return cls(groups, lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.01, max_grad_norm=max_grad_norm, **kw)


def _fused_state(opt, params):
    return {k: [opt.state[p][k] for p in params] for k in ('master', 'exp_avg', 'exp_avg_sq')}


def _sharded_state(opts):
    """Per-parameter fp32 state gathered from the shards of one layout (one optimizer per rank)."""
    o0 = opts[0]
    out = {k: [] for k in ('master', 'exp_avg', 'exp_avg_sq')}
    for j, (off, n) in enumerate(zip(o0.layout['offsets'], o0.layout['numels'])):
        for k in out:
            full = torch.empty(n, dtype=torch.float32, device='cuda')
            for o in opts:
                for jj, _, a, b in o.segments:
                    if jj == j:
                        full[a - off:b - off] = getattr(o, k)[a - o.rank * o.shard_size:b - o.rank * o.shard_size]
            out[k].append(full)
    return out


def _close_after_clip(a, b, what):
    """Bound with a binding clip: the gradient norms, added in different orders, agree to rel. 1e-5, and so do the
    clip coefficients.  An element of m moves with the coefficient times its gradient, one of v with its square, so
    their differences stay below 2e-5 / 4e-5 of the tensor's largest magnitude; Adam's m / sqrt(v) cancels the
    coefficient up to eps, so a master moves by at most lr x 1e-5 per step (1e-6 of the largest master); a bf16
    parameter may round to the neighbouring value (2^-7)."""
    rel = {'master': 1e-6, 'exp_avg': 2e-5, 'exp_avg_sq': 4e-5, 'param': 2 ** -7}[what]
    err = (a.float() - b.float()).abs().max().item()
    assert err <= rel * b.float().abs().max().item(), (what, err)


@pytest.mark.parametrize("h", [256, 320])
@pytest.mark.parametrize("max_grad_norm", [0.0, 1e4, 0.05])
def test_world1_train_step_equals_fused_adamw(h, max_grad_norm):
    """pretrain.train_step with ShardedFusedAdamW at world size 1; FusedAdamW steps a second model on the same
    gradients.  h = 320 puts tensor ends at offsets that are not multiples of 256."""
    from cogview_b200 import pretrain
    from cogview_b200.optim import FusedAdamW, ShardedFusedAdamW
    ms, gs = _model(h)
    mf, gf = _model(h)
    opt_s, opt_f = _opt(ShardedFusedAdamW, gs, max_grad_norm), _opt(FusedAdamW, gf, max_grad_norm)
    ps = [p for g in gs for p in g['params']]
    pf = [p for g in gf for p in g['params']]
    for step in range(4):
        loss, skipped, *_ = pretrain.train_step(_batch(seed=step), ms, opt_s)
        assert skipped == 0
        for p, q in zip(ps, pf):
            q.grad = p.grad.clone()
        opt_f.step()
        if max_grad_norm > 0:
            a, b = opt_s.last_grad_norm.item(), opt_f.last_grad_norm.item()
            assert abs(a - b) <= 1e-5 * b, (a, b)
            assert opt_f.last_step_skipped.item() == 0
        st_s, st_f = _sharded_state([opt_s]), _fused_state(opt_f, pf)
        if max_grad_norm != 0.05:
            for p, q in zip(ps, pf):
                assert torch.equal(p, q)
            for k in st_s:
                for a, b in zip(st_s[k], st_f[k]):
                    assert torch.equal(a, b.view(-1)), k
        else:
            assert opt_f.last_grad_norm.item() > 0.05     # the clip binds
            for p, q in zip(ps, pf):
                _close_after_clip(p, q, 'param')
            for k in st_s:
                for a, b in zip(st_s[k], st_f[k]):
                    _close_after_clip(a, b.view(-1), k)


def _grads_like(params, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return [(torch.randn(p.shape, generator=g, device='cuda') * 1e-2).bfloat16() for p in params]


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("max_grad_norm", [0.0, 0.05])
def test_virtual_shards_equal_fused_adamw(world, max_grad_norm):
    """Rank r's step of a world-size-N layout for r = 0..N-1 in one process on the same (averaged) gradients, the
    sum of squares added up in rank order and the parameters gathered by hand, against FusedAdamW."""
    from cogview_b200.optim import FusedAdamW, ShardedFusedAdamW
    h = 320
    mf, gf = _model(h)
    opt_f = _opt(FusedAdamW, gf, max_grad_norm)
    pf = [p for g in gf for p in g['params']]
    models, opts = [], []
    for r in range(world):
        m, g = _model(h)
        models.append([p for gg in g for p in gg['params']])
        opts.append(_opt(ShardedFusedAdamW, g, max_grad_norm, world_size=world, rank=r))
    assert any(o.layout['offsets'][j] < a or b < o.layout['offsets'][j] + o.layout['numels'][j]
               for o in opts for j, _, a, b in o.segments), "no tensor is split between shards"
    S = opts[0].shard_size
    for step in range(3):
        grads = _grads_like(pf, 100 + step)
        for q, g in zip(pf, grads):
            q.grad = g
        opt_f.step()
        for o, ps in zip(opts, models):
            o.zero_grad()
            for p, g in zip(ps, grads):
                p.grad.copy_(g)
        with torch.no_grad():
            tables = [o._prepare() for o in opts]
            if max_grad_norm > 0:
                total = torch.zeros(1, device='cuda')
                for o in opts:
                    total += o._scal[0:1]
                for o in opts:
                    o._scal[0:1].copy_(total)
            for o, t in zip(opts, tables):
                o._apply(t)
            for r, o in enumerate(opts):                  # the all-gather
                for o2 in opts:
                    if o2 is not o:
                        o2.flat_params[r * S:(r + 1) * S].copy_(o.flat_params[r * S:(r + 1) * S])
        st_s, st_f = _sharded_state(opts), _fused_state(opt_f, pf)
        for ps in models:
            for p, q in zip(ps, pf):
                if max_grad_norm == 0:
                    assert torch.equal(p, q)
                else:
                    _close_after_clip(p, q, 'param')
        for k in st_s:
            for a, b in zip(st_s[k], st_f[k]):
                if max_grad_norm == 0:
                    assert torch.equal(a, b.view(-1)), k
                else:
                    _close_after_clip(a, b.view(-1), k)
        if max_grad_norm > 0:
            a, b = opts[0].last_grad_norm.item(), opt_f.last_grad_norm.item()
            assert abs(a - b) <= 1e-5 * b and b > max_grad_norm, (a, b)


def test_gradient_views_survive_zero_grad_and_backward():
    from cogview_b200 import pretrain
    from cogview_b200.optim import ShardedFusedAdamW
    m, g = _model(256, ckpt=True)
    opt = _opt(ShardedFusedAdamW, g, 1.0)
    params = [p for gg in g for p in gg['params']]
    ptrs = [(p.data_ptr(), p.grad.data_ptr()) for p in params]
    base = opt.flat_grads.data_ptr()
    assert all(gp - base == pp - opt.flat_params.data_ptr() for pp, gp in ptrs)
    for step in range(2):
        pretrain.train_step(_batch(seed=step), m, opt, fused_loss=bool(step))
        assert [(p.data_ptr(), p.grad.data_ptr()) for p in params] == ptrs
        assert bool(opt.flat_grads.abs().sum() > 0)
    opt.zero_grad(set_to_none=True)
    assert [(p.data_ptr(), p.grad.data_ptr()) for p in params] == ptrs and not bool(opt.flat_grads.any())


def test_sharded_checkpoint_resumes_in_fused_adamw(tmp_path):
    """Two sharded steps, save_checkpoint (consolidated), load_checkpoint into FusedAdamW, two more steps: equal bit
    for bit to four FusedAdamW steps on the same gradients."""
    from cogview_b200 import checkpoint
    from cogview_b200.optim import FusedAdamW, ShardedFusedAdamW
    h = 320
    m_ref, g_ref = _model(h)
    ref = _opt(FusedAdamW, g_ref, 1e4)
    p_ref = [p for g in g_ref for p in g['params']]
    m_s, g_s = _model(h)
    sh = _opt(ShardedFusedAdamW, g_s, 1e4)
    p_s = [p for g in g_s for p in g['params']]
    grads = [_grads_like(p_ref, 200 + i) for i in range(4)]
    for i in range(4):
        for q, g in zip(p_ref, grads[i]):
            q.grad = g
        ref.step()
    for i in range(2):
        sh.zero_grad()
        for p, g in zip(p_s, grads[i]):
            p.grad.copy_(g)
        sh.step()
    checkpoint.save_checkpoint(2, m_s, sh, None, str(tmp_path))
    m_r, g_r = _model(h, seed=99)                 # other weights: the checkpoint must bring them back
    res = _opt(FusedAdamW, g_r, 1e4)
    assert checkpoint.load_checkpoint(m_r, res, None, str(tmp_path), no_load_rng=True) == 2
    p_r = [p for g in g_r for p in g['params']]
    for i in range(2, 4):
        for q, g in zip(p_r, grads[i]):
            q.grad = g
        res.step()
    for a, b in zip(p_r, p_ref):
        assert torch.equal(a, b)
    for k in ('master', 'exp_avg', 'exp_avg_sq'):
        for a, b in zip(_fused_state(res, p_r)[k], _fused_state(ref, p_ref)[k]):
            assert torch.equal(a, b), k
    assert res.state_dict()['applied_steps'] == ref.state_dict()['applied_steps'] == 4


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_worker(rank, world, port, out):
    import torch.distributed as dist
    from cogview_b200 import pretrain
    from cogview_b200.optim import ShardedFusedAdamW
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    m, g = _model(320)
    opt = _opt(ShardedFusedAdamW, g, 1.0)
    for step in range(3):
        loss, skipped, *_ = pretrain.train_step(_batch(seed=10 * step + rank), m, opt)
        assert skipped == 0
    flat = opt.flat_params.clone()
    every = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every), "ranks hold different parameters"
    out[rank] = [p.detach().cpu() for gg in g for p in gg['params']]
    dist.destroy_process_group()


def test_two_ranks_nccl_match_single_process():
    """Two ranks under NCCL, each on its own batch, against one process stepping FusedAdamW on the average of the
    two batches' gradients.  The reduce-scatter averages in bf16: parameters agree within a few bf16 ulp."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs, %d visible" % torch.cuda.device_count())
    import torch.multiprocessing as mp
    from cogview_b200 import pretrain
    from cogview_b200.optim import FusedAdamW
    world = 2
    out = mp.get_context('spawn').Manager().dict()
    mp.spawn(_nccl_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    m, g = _model(320)
    opt = _opt(FusedAdamW, g, 1.0)
    params = [p for gg in g for p in gg['params']]
    for step in range(3):
        acc = None
        for r in range(world):
            for p in params:
                p.grad = None
            loss, *_ = pretrain.forward_step(_batch(seed=10 * step + r), m)
            loss.backward()
            gr = [p.grad.float() for p in params]
            acc = gr if acc is None else [a + b for a, b in zip(acc, gr)]
        for p, a in zip(params, acc):
            p.grad = (a / world).bfloat16()
        opt.step()
    for p, q in zip(params, out[0]):
        d = (p.detach().cpu().float() - q.float()).abs().max().item()
        assert d <= 4 * 2 ** -8 * max(q.float().abs().max().item(), 1e-3), d
