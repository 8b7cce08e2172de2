"""ShardedFusedAdamW (cogview_b200/optim.py, ZeRO stage 1) at world size 2 over gloo on the CPU.  The collectives,
the flat layout, the segment tables and the checkpoint logic are the real ones; only the three optim.cu launches
(cv_sumsq_bf16_multi, cv_clip_coef, cv_adamw_step_multi) are replaced by a torch stand-in that follows the same
cv_adamw_entry table, reading and writing through its pointers."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

LR = (1e-2, 3e-2)
WD = (0.1, 0.0)
B1, B2, EPS = 0.9, 0.99, 1e-6


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _at(addr, n, dtype):
    """A CPU tensor over n elements at address addr (bf16 or fp32), sharing that memory."""
    arr = np.ctypeslib.as_array(((ctypes.c_uint16 if dtype == torch.bfloat16 else ctypes.c_float) * n).from_address(addr))
    t = torch.from_numpy(arr)
    return t.view(torch.bfloat16) if dtype == torch.bfloat16 else t


class TorchKernels:
    """Stand-in of optim._Kernels on CPU tensors: the same table, the same arithmetic as csrc/optim.cu (in fp32)."""

    def __init__(self):
        self.tables = []

    def stage(self, n, dev):
        from cogview_b200.optim import _ENTRY
        self.rec = np.zeros(n, dtype=_ENTRY)
        return self.rec

    def upload(self):
        self.tables.append(self.rec.copy())
        return self.tables[-1]

    def sumsq(self, table, count, out):
        assert len(table) == count
        for e in table:
            assert e['grad'] % 16 == 0
            out += _at(int(e['grad']), int(e['n']), torch.bfloat16).float().square().sum()

    def clip_coef(self, sumsq, max_norm, coef, norm_out, state):
        nrm = sumsq.sqrt()
        norm_out.copy_(nrm)
        bad = not bool(torch.isfinite(nrm))
        c = max_norm / (float(nrm) + 1e-6)
        coef.fill_(0.0 if bad else min(c, 1.0))
        state[0] = int(bad)
        if not bad:
            state[1] += 1

    def adamw(self, table, count, b1, b2, eps, coef, state):
        if state is not None and int(state[0]):
            return
        gs = 1.0 if coef is None else float(coef)
        for e in table[:count]:
            n = int(e['n'])
            for k in ('param', 'grad'):
                assert e[k] % 16 == 0
            for k in ('master', 'm', 'v'):
                assert e[k] % 32 == 0
            p, g = _at(int(e['param']), n, torch.bfloat16), _at(int(e['grad']), n, torch.bfloat16)
            w, m, v = (_at(int(e[k]), n, torch.float32) for k in ('master', 'm', 'v'))
            bc1, bc2 = float(e['bc1']), float(e['bc2'])
            if state is not None:
                bc1, bc2 = 1.0 - b1 ** int(state[1]), 1.0 - b2 ** int(state[1])
            gf = g.float() * gs
            m.mul_(b1).add_((1 - b1) * gf)
            v.mul_(b2).add_((1 - b2) * gf * gf)
            w.sub_(float(e['lr']) * ((m / bc1) / ((v / bc2).sqrt() + eps) + float(e['wd']) * w))
            p.copy_(w.to(torch.bfloat16))


def _model(seed):
    """Parameters of awkward sizes (none a multiple of 8) in the two weight-decay groups of the GPT-2 model."""
    from cogview_b200.model import gpt2_get_params_for_weight_decay_optimization
    torch.manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Linear(7, 5), torch.nn.LayerNorm(5), torch.nn.Linear(5, 13),
                              torch.nn.Embedding(11, 3)).bfloat16()
    groups = gpt2_get_params_for_weight_decay_optimization(net)
    for g, lr, wd in zip(groups, LR, WD):
        g['lr'], g['weight_decay'] = lr, wd
    return net, groups


def _grads(params, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(p.shape, generator=g).bfloat16() for p in params]


def _worker(rank, world, port, tmp, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cogview_b200.optim import FusedAdamW, ShardedFusedAdamW
    net, groups = _model(seed=10 + rank)              # different init per rank: rank 0's is broadcast
    groups_of = [gi for gi, g in enumerate(groups) for _ in g['params']]
    opt = ShardedFusedAdamW(groups, lr=1.0, betas=(B1, B2), eps=EPS, max_grad_norm=1.0)
    opt._kern = TorchKernels()
    params = [p for g in groups for p in g['params']]

    # flat layout: aligned starts, padded total, shards covering every element exactly once
    L = opt.layout
    assert L['world_size'] == world and L['padded_total'] % (8 * world) == 0
    assert all(o % 8 == 0 for o in L['offsets'])
    assert all(b >= a + n for a, n, b in zip(L['offsets'], L['numels'], L['offsets'][1:] + [L['padded_total']]))
    for p, o, n in zip(params, L['offsets'], L['numels']):
        assert p.data_ptr() == opt.flat_params.data_ptr() + 2 * o and p.numel() == n
        assert p.grad.data_ptr() == opt.flat_grads.data_ptr() + 2 * o
    S = opt.shard_size
    assert S * world == L['padded_total'] and opt.master.numel() == S
    covered = torch.zeros(L['padded_total'], dtype=torch.int32)
    segs = [None] * world
    dist.all_gather_object(segs, opt.segments)
    for q, ss in enumerate(segs):
        for j, gi, a, b in ss:
            assert q * S <= a < b <= (q + 1) * S and gi == groups_of[j]
            assert L['offsets'][j] <= a and b <= L['offsets'][j] + L['numels'][j]
            covered[a:b] += 1
    want = torch.zeros_like(covered)
    for o, n in zip(L['offsets'], L['numels']):
        want[o:o + n] = 1
    assert torch.equal(covered, want), "every parameter element in exactly one shard segment"
    assert any(L['offsets'][j] < a or b < L['offsets'][j] + L['numels'][j] for ss in segs for j, _, a, b in ss), \
        "the layout must split a tensor between the shards"
    # parameters were broadcast from rank 0
    flat = [torch.zeros_like(opt.flat_params) for _ in range(world)]
    dist.all_gather(flat, opt.flat_params)
    assert torch.equal(flat[0], flat[1])
    params0 = [p.detach().clone() for p in params]

    # a real backward accumulates into the flat buffer's views
    opt.zero_grad(set_to_none=True)
    net[0](torch.ones(2, 7, dtype=torch.bfloat16)).sum().backward()
    assert net[0].weight.grad.data_ptr() == opt.flat_grads.data_ptr() + 2 * L['offsets'][params.index(net[0].weight)]
    assert bool((net[0].weight.grad == 2).all())

    # steps on rank-dependent gradients == single-process AdamW on their average, identical on both ranks
    steps = 3
    grad_sets = [[_grads(params, 100 * t + q) for q in range(world)] for t in range(steps)]
    for t in range(steps):
        opt.zero_grad()
        for p, g in zip(params, grad_sets[t][rank]):
            p.grad.copy_(g)
        opt.step()
        assert int(opt.last_step_skipped) == 0
        # the table of this step: pointers into the shard, the segment's group's lr and weight decay
        rec = opt._kern.tables[-1]
        assert len(rec) == len(opt.segments)
        for e, (j, gi, a, b) in zip(rec, opt.segments):
            assert e['param'] == opt.flat_params.data_ptr() + 2 * a and e['grad'] == opt.flat_grads.data_ptr() + 2 * a
            assert e['master'] == opt.master.data_ptr() + 4 * (a - rank * S) and e['n'] == b - a
            assert e['lr'] == np.float32(LR[gi]) and e['wd'] == np.float32(WD[gi])
    flat = [torch.zeros_like(opt.flat_params) for _ in range(world)]
    dist.all_gather(flat, opt.flat_params)
    assert torch.equal(flat[0], flat[1]), "ranks hold different parameters"
    ref_w, ref_m, ref_v = _reference_steps(params0, grad_sets, groups_of, 1.0)
    cons = opt.consolidated_state_dict()
    if rank == 0:
        for i, p in enumerate(params):
            st = cons['state'][i]
            assert st['step'] == steps and st['master'].shape == p.shape and st['master'].dtype == torch.float32
            assert torch.allclose(st['master'].double(), ref_w[i], rtol=1e-5, atol=1e-6), i
            assert torch.allclose(st['exp_avg'].double(), ref_m[i], rtol=1e-4, atol=1e-7), i
            assert torch.allclose(st['exp_avg_sq'].double(), ref_v[i], rtol=1e-4, atol=1e-9), i
            assert torch.equal(p.detach(), st['master'].to(torch.bfloat16)), i
        assert cons['applied_steps'] == steps and [g['lr'] for g in cons['param_groups']] == list(LR)
    else:
        assert cons is None

    # a non-finite gradient on one rank skips the step on both
    before = opt.flat_params.clone()
    m_before = opt.exp_avg.clone()
    opt.zero_grad()
    for p, g in zip(params, _grads(params, 999 + rank)):
        p.grad.copy_(g)
    if rank == 1:
        params[-1].grad.view(-1)[0] = float('inf')
    opt.step()
    assert int(opt.last_step_skipped) == 1
    assert torch.equal(opt.flat_params, before) and torch.equal(opt.exp_avg, m_before)
    assert opt._applied_steps() == steps

    # state_dict round trip, layout mismatch, consolidated <-> FusedAdamW
    sd = opt.state_dict()
    path = os.path.join(tmp, "shard%d.pt" % rank)
    torch.save(sd, path)
    net2, groups2 = _model(seed=10)
    opt2 = ShardedFusedAdamW(groups2, lr=1.0, betas=(B1, B2), eps=EPS, max_grad_norm=1.0)
    opt2.load_state_dict(torch.load(path, weights_only=False))
    for k in ('master', 'exp_avg', 'exp_avg_sq'):
        assert torch.equal(getattr(opt2, k), getattr(opt, k)), k
    assert opt2._step == steps + 1 and opt2._applied == steps
    assert [g['lr'] for g in opt2.param_groups] == list(LR)
    other = dict(sd, rank=1 - rank)
    with pytest.raises(ValueError):
        opt2.load_state_dict(other)
    single = ShardedFusedAdamW(_model(seed=10)[1], lr=1.0, world_size=1, rank=0)
    with pytest.raises(ValueError):
        single.load_state_dict(sd)
    cons = opt.consolidated_state_dict()
    if rank == 0:
        torch.save(cons, os.path.join(tmp, "consolidated.pt"))
    dist.barrier()
    cons = torch.load(os.path.join(tmp, "consolidated.pt"), weights_only=False)
    # into a plain FusedAdamW (one process, the whole state)
    net3, groups3 = _model(seed=10)
    fused = FusedAdamW(groups3, lr=1.0, betas=(B1, B2), eps=EPS, max_grad_norm=1.0)
    fused.load_state_dict(cons)
    assert fused._applied == steps
    for i, p in enumerate(p for g in groups3 for p in g['params']):
        assert fused.state[p]['step'] == steps + 1
        assert torch.equal(fused.state[p]['master'], cons['state'][i]['master'])
    # and back into shards of another world size: each of 3 virtual ranks takes its range
    for r in range(3):
        sh = ShardedFusedAdamW(_model(seed=10)[1], lr=1.0, world_size=3, rank=r)
        sh.load_state_dict(fused.state_dict())
        back = dict(fused.state_dict())
        for j, gi, a, b in sh.segments:
            o = sh.layout['offsets'][j]
            for k in ('master', 'exp_avg', 'exp_avg_sq'):
                want = back['state'][j][k].reshape(-1)[a - o:b - o]
                assert torch.equal(getattr(sh, k)[a - r * sh.shard_size:b - r * sh.shard_size], want), (r, j, k)
        assert sh._step == steps + 1 and sh._applied == steps
    # into the same world size through load_state_dict: the shards come back bit for bit
    net4, groups4 = _model(seed=10)
    opt4 = ShardedFusedAdamW(groups4, lr=1.0, betas=(B1, B2), eps=EPS, max_grad_norm=1.0)
    opt4.load_state_dict(cons)
    for k in ('master', 'exp_avg', 'exp_avg_sq'):
        assert torch.equal(getattr(opt4, k), getattr(opt, k)), k
    out[rank] = 1
    dist.barrier()
    dist.destroy_process_group()


def _reference_steps(params0, grad_sets, groups_of, max_norm):
    """Single-process AdamW in float64 on the averaged gradients (grad_sets[step][rank]), with the same clipping."""
    w = [p.double() for p in params0]
    m = [torch.zeros_like(x) for x in w]
    v = [torch.zeros_like(x) for x in w]
    for t, per_rank in enumerate(grad_sets, start=1):
        avg = [(sum(gs[i].float() for gs in per_rank) / len(per_rank)).bfloat16().double() for i in range(len(w))]
        nrm = float(torch.sqrt(sum((g * g).sum() for g in avg)))
        c = min(1.0, max_norm / (nrm + 1e-6))
        for i, g in enumerate(avg):
            lr, wd = LR[groups_of[i]], WD[groups_of[i]]
            g = g * c
            m[i] = B1 * m[i] + (1 - B1) * g
            v[i] = B2 * v[i] + (1 - B2) * g * g
            w[i] = w[i] - lr * ((m[i] / (1 - B1 ** t)) / (torch.sqrt(v[i] / (1 - B2 ** t)) + EPS) + wd * w[i])
    return w, m, v


def test_sharded_adamw_world2(tmp_path):
    world = 2
    mgr = mp.get_context('spawn').Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), out), nprocs=world, join=True)
    assert sorted(out.keys()) == [0, 1]


def test_zero_grad_keeps_views_and_step_refuses_detached_gradients():
    from cogview_b200.optim import ShardedFusedAdamW
    net, groups = _model(seed=1)
    opt = ShardedFusedAdamW(groups, lr=1e-3)
    opt._kern = TorchKernels()
    ptrs = [p.grad.data_ptr() for p in net.parameters()]
    for p in net.parameters():
        p.grad.fill_(1.0)
    opt.zero_grad(set_to_none=True)
    assert [p.grad.data_ptr() for p in net.parameters()] == ptrs
    assert not bool(opt.flat_grads.any())
    net[0].weight.grad = None
    opt.zero_grad()
    assert net[0].weight.grad.data_ptr() == ptrs[0]
    net[0].weight.grad = torch.zeros_like(net[0].weight)
    with pytest.raises(RuntimeError):
        opt.step()
