"""Fused AdamW for bf16 models with fp32 master weights — the CUDA replacement of the reference's
FP16_Optimizer + apex FusedAdam + mpu.clip_grad_norm sequence (pretrain_gpt2.py:110-158, :380-389, :437-444;
fp16/fp16.py:291-310, :399-453; mpu/grads.py:28-74).  bf16 needs no loss scaling, so the dynamic loss scaler
disappears; the NaN/inf guard of train_step (pretrain_gpt2.py:415-417) stays with the caller.

The clip coefficient is computed on the device (cv_sumsq_bf16_multi + cv_clip_coef) and consumed by
cv_adamw_step_multi through a device pointer, so a step never synchronises with the host.  The whole parameter
list is one table (cv_adamw_entry, include/cogview_b200.h) -> three launches per step instead of two per tensor."""
import numpy as np
import torch

from ._lib import check, lib, ptr, stream_ptr


_ENTRY = np.dtype([('param', '<u8'), ('grad', '<u8'), ('master', '<u8'), ('m', '<u8'), ('v', '<u8'), ('n', '<i8'),
                   ('lr', '<f4'), ('wd', '<f4'), ('bc1', '<f4'), ('bc2', '<f4')])   # = cv_adamw_entry, 64 bytes


class _Kernels:
    """The csrc/optim.cu launches of one optimizer step over a cv_adamw_entry table.  The table is staged in pinned
    host memory, double-buffered because the previous step's copy may still be in flight, and copied to the device
    asynchronously, so a step never waits for the host."""

    def __init__(self):
        self._bufs = None            # (pinned host staging x2, device table), reallocated when the entry count changes
        self._copied = [None, None]  # CUDA event recorded after the async copy out of each staging buffer
        self._flip = 0

    def stage(self, n, dev):
        """The host records (numpy, dtype _ENTRY) of the next table, n entries on device dev."""
        if self._bufs is None or self._bufs[2].numel() != n * 64 or self._bufs[2].device != dev:
            host = [torch.empty(n * 64, dtype=torch.uint8).pin_memory() for _ in range(2)]
            self._bufs = (host[0], host[1], torch.empty(n * 64, dtype=torch.uint8, device=dev))
            self._copied = [None, None]
        self._flip ^= 1
        if self._copied[self._flip] is not None:          # the copy issued two steps ago has long finished; make sure
            self._copied[self._flip].synchronize()
        return self._bufs[self._flip].numpy().view(_ENTRY)

    def upload(self):
        """Copies the staged records to the device table and returns it."""
        self._bufs[2].copy_(self._bufs[self._flip], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._copied[self._flip] = ev
        return self._bufs[2]

    def sumsq(self, table, count, out):
        check(lib().cv_sumsq_bf16_multi(ptr(table), count, ptr(out), stream_ptr()), "cv_sumsq_bf16_multi")

    def clip_coef(self, sumsq, max_norm, coef, norm_out, state):
        check(lib().cv_clip_coef(ptr(sumsq), max_norm, ptr(coef), ptr(norm_out), ptr(state), stream_ptr()),
              "cv_clip_coef")

    def adamw(self, table, count, beta1, beta2, eps, coef, state):
        check(lib().cv_adamw_step_multi(ptr(table), count, float(beta1), float(beta2), float(eps), ptr(coef), 1.0,
                                        ptr(state), stream_ptr()), "cv_adamw_step_multi")


class FusedAdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_grad_norm=0.0):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.max_grad_norm = float(max_grad_norm)
        self._scal = None
        self._kern = _Kernels()      # table staging + the three launches of a step
        self.last_grad_norm = None   # device tensor (1,) after step() when clipping is on
        self._state = None           # device int32 [2]: [0] last step skipped (non-finite gradient norm), [1] applied steps
        self._applied = 0            # applied steps restored from a checkpoint (seeds the device counter)

    _FP32_STATE = ('master', 'exp_avg', 'exp_avg_sq')

    @property
    def last_step_skipped(self):
        """Device int32 view (1,) — 1 when the last step() was skipped because the gradient norm was inf/NaN (the
        overflow branch of FP16_Optimizer.step, fp16/fp16.py:399-420), or None before the first clipped step."""
        return None if self._state is None else self._state[0:1]

    def state_dict(self):
        sd = super().state_dict()
        if self._state is not None:
            self._applied = int(self._state[1].item())
        sd['applied_steps'] = self._applied
        return sd

    def load_state_dict(self, state_dict):
        """torch.optim.Optimizer.load_state_dict casts every floating-point state tensor to the PARAMETER dtype (bf16
        here), which would halve the fp32 masters and moments the kernels address as float*.  Restore them from the
        incoming dict in fp32 after the generic load."""
        state_dict = dict(state_dict)
        self._applied = int(state_dict.pop('applied_steps', 0))
        if 'state' not in state_dict or 'param_groups' not in state_dict or any(
                'params' not in g for g in state_dict['param_groups']):
            raise ValueError('FusedAdamW.load_state_dict: not a torch.optim state_dict (a reference FP16_Optimizer / '
                             'DeepSpeed optimizer entry cannot be loaded: resume with no_load_optim)')
        super().load_state_dict(state_dict)
        saved_ids = [i for g in state_dict['param_groups'] for i in g['params']]
        params = [p for g in self.param_groups for p in g['params']]
        for idx, p in zip(saved_ids, params):
            src = state_dict['state'].get(idx)
            if src is None:
                continue
            st = self.state[p]
            for k in self._FP32_STATE:
                if k in src:
                    st[k] = src[k].detach().to(device=p.device, dtype=torch.float32).contiguous().clone()
            if 'step' in src:
                st['step'] = int(src['step'])
            if not self._applied:
                self._applied = int(st.get('step', 0))
        self._state = None

    def _table(self, plist, dev):
        """Fills the device-resident cv_adamw_entry table for this step (gradient pointers may move between steps)."""
        rec = self._kern.stage(len(plist), dev)
        for i, (group, p) in enumerate(plist):
            st = self._state_for(p)
            for k in self._FP32_STATE:
                t = st[k]
                assert t.dtype == torch.float32 and t.numel() == p.numel() and t.is_contiguous() and t.device == p.device, \
                    "FusedAdamW state '%s' must be a contiguous fp32 tensor of the parameter's size" % k
            st['step'] += 1
            b1, b2 = group['betas']
            rec[i] = (p.data_ptr(), p.grad.data_ptr(), st['master'].data_ptr(), st['exp_avg'].data_ptr(),
                      st['exp_avg_sq'].data_ptr(), p.numel(), group['lr'], group['weight_decay'],
                      1.0 - b1 ** st['step'], 1.0 - b2 ** st['step'])
        return self._kern.upload()

    def _state_for(self, p):
        st = self.state[p]
        if not st:
            st['step'] = 0
            st['master'] = p.detach().float().clone()
            st['exp_avg'] = torch.zeros_like(st['master'])
            st['exp_avg_sq'] = torch.zeros_like(st['master'])
        return st

    @torch.no_grad()
    def step(self, closure=None):
        assert closure is None
        plist = [(g, p) for g in self.param_groups for p in g['params'] if p.grad is not None]
        if not plist:
            return None
        dev = plist[0][1].device
        for group, p in plist:
            assert p.dtype == torch.bfloat16 and p.is_contiguous(), "FusedAdamW expects contiguous bf16 parameters"
            g = p.grad
            assert g.dtype == torch.bfloat16 and g.is_contiguous(), "FusedAdamW expects contiguous bf16 gradients"
        assert len({(g['betas'], g['eps']) for g, _ in plist}) == 1, "betas / eps must be the same for all groups"
        b1, b2 = plist[0][0]['betas']
        eps = plist[0][0]['eps']
        table = self._table(plist, dev)
        coef = None
        if self.max_grad_norm > 0:
            self._clip_buffers(dev)
            self._kern.sumsq(table, len(plist), self._scal[0:1])
            coef = self._clip()
        self._kern.adamw(table, len(plist), b1, b2, eps, coef, self._state if self.max_grad_norm > 0 else None)
        return None

    def _clip_buffers(self, dev):
        """Zeroed sum-of-squares accumulator (self._scal = [sumsq, coef, norm]) and the skip / applied-step state."""
        if self._scal is None or self._scal.device != dev:
            self._scal = torch.zeros(3, dtype=torch.float32, device=dev)
        if self._state is None or self._state.device != dev:
            self._state = torch.tensor([0, self._applied], dtype=torch.int32, device=dev)
        self._scal.zero_()

    def _clip(self):
        """Clip coefficient (device scalar) from the accumulated sum of squares; sets last_grad_norm and the skip flag."""
        self._kern.clip_coef(self._scal[0:1], self.max_grad_norm, self._scal[1:2], self._scal[2:3], self._state)
        self.last_grad_norm = self._scal[2:3]
        return self._scal[1:2]


_ALIGN = 8          # elements: a bf16 segment start is 16-byte aligned, an fp32 one 32-byte aligned


def _round_up(x, m):
    return (x + m - 1) // m * m


class ShardedFusedAdamW(FusedAdamW):
    """FusedAdamW with the fp32 state sharded over the data-parallel ranks (ZeRO stage 1): each rank keeps the master
    weights and both moments of 1 / world of the parameters.  The same update and the same global-norm clipping as
    FusedAdamW; the reference's DeepSpeed setting "zero_optimization": {"stage": 1, "reduce_scatter": true}.

    Flat layout.  At construction every parameter is copied into one flat bf16 buffer and `p.data` becomes a view
    of it; `p.grad` becomes a view of a flat bf16 gradient buffer of the same layout, into which the backward
    accumulates in place.  Every tensor starts at a multiple of 8 elements and the total is padded to a multiple of
    8 x world, so every segment and every shard boundary is 16-byte aligned for the vector accesses of csrc/optim.cu.
    Rank r owns the range [r S, (r + 1) S) of S = total / world elements.  Build the model, move it to its device
    and cast it to bf16 before constructing the optimizer; parameters replaced afterwards (.to(), .cuda()) would
    leave the flat buffers.  Model caches keyed on parameter pointers (the decode runner's captured graphs) see the
    new pointers and rebuild.

    step(), without a host synchronisation:
      1. reduce-scatter (average) of the flat gradients: each rank receives the averaged gradients of its range.
         This replaces DDP's all-reduce: do not wrap the model in DDP;
      2. sum of squares of the owned gradients (cv_sumsq_bf16_multi), all-reduced over the ranks;
      3. clip coefficient (cv_clip_coef): every rank sees the same norm, so a non-finite norm skips the step on all
         of them together (last_step_skipped);
      4. AdamW (cv_adamw_step_multi) over one table entry per piece of a tensor in the owned range, with that
         tensor's group's lr and weight decay;
      5. all-gather of the flat parameters.

    Checkpoints.  state_dict() / load_state_dict() hold this rank's shard and the layout it belongs to (world size,
    padded offsets); load_state_dict() of a different layout raises ValueError.  consolidated_state_dict() (called
    on every rank) assembles FusedAdamW.state_dict()'s form on rank 0, and load_state_dict() of that form builds this
    rank's shard from it, so a run moves between sharded and unsharded training and between world sizes.

    `world_size` / `rank` build one rank's shard of a layout without a process group (no collectives are issued);
    by default they are those of `process_group` (the default group when torch.distributed is initialized, else 1
    and 0).  Rank 0's parameters are broadcast to the other ranks at construction."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_grad_norm=0.0,
                 process_group=None, *, world_size=None, rank=None):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, max_grad_norm=max_grad_norm)
        dist = torch.distributed
        self.process_group = process_group
        self._collective = world_size is None and rank is None and dist.is_available() and dist.is_initialized()
        if self._collective:
            world_size, rank = dist.get_world_size(process_group), dist.get_rank(process_group)
        self.world_size = 1 if world_size is None else int(world_size)
        self.rank = 0 if rank is None else int(rank)
        if not 0 <= self.rank < self.world_size:
            raise ValueError('rank %d outside world size %d' % (self.rank, self.world_size))
        self._collective = self._collective and self.world_size > 1
        self._params = [p for g in self.param_groups for p in g['params']]
        if not self._params:
            raise ValueError('ShardedFusedAdamW got no parameters')
        dev = self._params[0].device
        for p in self._params:
            if p.dtype != torch.bfloat16 or p.device != dev:
                raise ValueError('ShardedFusedAdamW expects bf16 parameters on one device')
        offsets, o = [], 0
        for p in self._params:
            offsets.append(o)
            o += _round_up(p.numel(), _ALIGN)
        total = _round_up(o, _ALIGN * self.world_size)
        self.layout = dict(world_size=self.world_size, offsets=offsets, numels=[p.numel() for p in self._params],
                           padded_total=total)
        self.shard_size = S = total // self.world_size
        self.flat_params = torch.zeros(total, dtype=torch.bfloat16, device=dev)
        self.flat_grads = torch.zeros(total, dtype=torch.bfloat16, device=dev)
        self._grad_views = []
        with torch.no_grad():
            for p, o in zip(self._params, offsets):
                n = p.numel()
                self.flat_params[o:o + n].copy_(p.reshape(-1))
                p.data = self.flat_params[o:o + n].view(p.shape)
                p.grad = self.flat_grads[o:o + n].view(p.shape)
                self._grad_views.append(p.grad)
        if self._collective:
            dist.broadcast(self.flat_params, src=self._global_rank(0), group=process_group)
        lo = self.rank * S
        self.master = torch.zeros(S, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros_like(self.master)
        self.exp_avg_sq = torch.zeros_like(self.master)
        self._master_set = False     # the masters are read from the parameters at the first step, as FusedAdamW does
        self._step = 0               # step() calls (FusedAdamW's per-tensor 'step')
        # segments: (parameter index, group index, first, last + 1) in flat-buffer elements, clipped to the shard
        group_of = [gi for gi, g in enumerate(self.param_groups) for _ in g['params']]
        self.segments = []
        for j, (o, n) in enumerate(zip(offsets, self.layout['numels'])):
            a, b = max(o, lo), min(o + n, lo + S)
            if a < b:
                self.segments.append((j, group_of[j], a, b))
        first = np.array([s[2] for s in self.segments], dtype=np.int64)
        self._seg_group = [s[1] for s in self.segments]
        self._seg_ptrs = (self.flat_params.data_ptr() + 2 * first, self.flat_grads.data_ptr() + 2 * first,
                          self.master.data_ptr() + 4 * (first - lo), self.exp_avg.data_ptr() + 4 * (first - lo),
                          self.exp_avg_sq.data_ptr() + 4 * (first - lo),
                          np.array([s[3] - s[2] for s in self.segments], dtype=np.int64))

    def _global_rank(self, group_rank):
        pg = self.process_group
        return group_rank if pg is None else torch.distributed.get_global_rank(pg, group_rank)

    def _shard(self, flat):
        return flat[self.rank * self.shard_size:(self.rank + 1) * self.shard_size]

    def zero_grad(self, set_to_none=True):
        """Zeroes the flat gradient buffer in place and keeps every `p.grad` a view of it.  `set_to_none` is ignored:
        a gradient set to None would be re-created outside the buffer by the next backward, and the step would not
        see it.  A `p.grad` replaced or set to None by the caller is re-attached to its view."""
        self.flat_grads.zero_()
        for p, g in zip(self._params, self._grad_views):
            if p.grad is None or p.grad.data_ptr() != g.data_ptr():
                p.grad = g

    @torch.no_grad()
    def step(self, closure=None):
        assert closure is None
        for p, g in zip(self._params, self._grad_views):
            if p.grad is None or p.grad.data_ptr() != g.data_ptr() or \
                    p.data_ptr() - self.flat_params.data_ptr() != g.data_ptr() - self.flat_grads.data_ptr():
                raise RuntimeError('ShardedFusedAdamW: a parameter or its gradient is no longer a view of the flat '
                                   'buffers (p.grad replaced, or the model moved / cast after the optimizer was built); '
                                   'call zero_grad() of this optimizer before the backward')
        if self._collective:
            torch.distributed.reduce_scatter_tensor(self._shard(self.flat_grads), self.flat_grads,
                                                    op=torch.distributed.ReduceOp.AVG, group=self.process_group)
        table = self._prepare()
        if self.max_grad_norm > 0 and self._collective:
            torch.distributed.all_reduce(self._scal[0:1], group=self.process_group)
        self._apply(table)
        if self._collective:
            torch.distributed.all_gather_into_tensor(self.flat_params, self._shard(self.flat_params),
                                                     group=self.process_group)
        return None

    def _prepare(self):
        """Steps 2 and 4's set-up on this rank: the segment table of this step, and (clipping on) the sum of squares
        of the owned gradients in self._scal[0], not yet summed over the ranks."""
        assert len({(g['betas'], g['eps']) for g in self.param_groups}) == 1, "betas / eps must be the same for all groups"
        dev = self.flat_params.device
        if not self._master_set:
            self.master.copy_(self._shard(self.flat_params))
            self._master_set = True
        self._step += 1
        b1, b2 = self.param_groups[0]['betas']
        table = None
        if self.segments:
            rec = self._kern.stage(len(self.segments), dev)
            for k, a in zip(('param', 'grad', 'master', 'm', 'v', 'n'), self._seg_ptrs):
                rec[k] = a
            rec['lr'] = [self.param_groups[gi]['lr'] for gi in self._seg_group]
            rec['wd'] = [self.param_groups[gi]['weight_decay'] for gi in self._seg_group]
            rec['bc1'] = 1.0 - b1 ** self._step
            rec['bc2'] = 1.0 - b2 ** self._step
            table = self._kern.upload()
        if self.max_grad_norm > 0:
            self._clip_buffers(dev)
            if table is not None:
                self._kern.sumsq(table, len(self.segments), self._scal[0:1])
        return table

    def _apply(self, table):
        """Steps 3 and 4 on this rank, once self._scal[0] holds the global sum of squares."""
        coef = self._clip() if self.max_grad_norm > 0 else None
        if table is not None:
            b1, b2 = self.param_groups[0]['betas']
            self._kern.adamw(table, len(self.segments), b1, b2, self.param_groups[0]['eps'], coef,
                             self._state if self.max_grad_norm > 0 else None)

    # -- checkpoints ---------------------------------------------------------------------------------------------
    def _hyper(self):
        return [{k: v for k, v in g.items() if k != 'params'} for g in self.param_groups]

    def _set_hyper(self, groups):
        if len(groups) != len(self.param_groups):
            raise ValueError('state_dict has %d param groups, the optimizer %d' % (len(groups), len(self.param_groups)))
        for g, sg in zip(self.param_groups, groups):
            g.update({k: v for k, v in sg.items() if k != 'params'})

    def _applied_steps(self):
        if self._state is not None:
            self._applied = int(self._state[1].item())
        return self._applied

    def state_dict(self):
        """This rank's shard: {'zero_layout', 'rank', 'param_groups' (hyper-parameters), 'step', 'applied_steps',
        'master', 'exp_avg', 'exp_avg_sq' (fp32 [S])}."""
        return {'zero_layout': dict(self.layout), 'rank': self.rank, 'param_groups': self._hyper(), 'step': self._step,
                'applied_steps': self._applied_steps(), 'master': self.master, 'exp_avg': self.exp_avg,
                'exp_avg_sq': self.exp_avg_sq}

    def load_state_dict(self, state_dict):
        """Loads a shard written by state_dict() under the same layout and rank (ValueError otherwise), or a
        FusedAdamW.state_dict() / consolidated_state_dict(), from which this rank's shard is taken."""
        if 'zero_layout' not in state_dict:
            return self._load_consolidated(state_dict)
        if state_dict['zero_layout'] != self.layout or state_dict['rank'] != self.rank:
            raise ValueError('ShardedFusedAdamW.load_state_dict: the shard was written for rank %d of layout %s, this '
                             'is rank %d of world size %d with another layout; load a consolidated_state_dict() instead'
                             % (state_dict['rank'], {k: v for k, v in state_dict['zero_layout'].items()
                                                     if k != 'offsets'}, self.rank, self.world_size))
        self._set_hyper(state_dict['param_groups'])
        for k in self._FP32_STATE:
            getattr(self, k).copy_(state_dict[k])
        self._master_set = True
        self._step = int(state_dict['step'])
        self._applied = int(state_dict['applied_steps'])
        self._state = None

    def _load_consolidated(self, state_dict):
        if 'state' not in state_dict or 'param_groups' not in state_dict or any(
                'params' not in g for g in state_dict['param_groups']):
            raise ValueError('ShardedFusedAdamW.load_state_dict: neither a shard nor a FusedAdamW state_dict')
        saved_ids = [i for g in state_dict['param_groups'] for i in g['params']]
        if len(saved_ids) != len(self._params):
            raise ValueError('state_dict holds %d parameters, the optimizer %d' % (len(saved_ids), len(self._params)))
        self._set_hyper(state_dict['param_groups'])
        lo, S = self.rank * self.shard_size, self.shard_size
        self.master.copy_(self._shard(self.flat_params))
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        step = 0
        for j, idx in enumerate(saved_ids):
            src = state_dict['state'].get(idx)
            if src is None:
                continue
            o, n = self.layout['offsets'][j], self.layout['numels'][j]
            a, b = max(o, lo), min(o + n, lo + S)
            for k in self._FP32_STATE:
                if k not in src:
                    continue
                if src[k].numel() != n:
                    raise ValueError("state '%s' of parameter %d has %d elements, the parameter %d"
                                     % (k, j, src[k].numel(), n))
                if a < b:
                    getattr(self, k)[a - lo:b - lo].copy_(src[k].detach().reshape(-1)[a - o:b - o])
            step = max(step, int(src.get('step', 0)))
        self._master_set = True
        self._step = step
        self._applied = int(state_dict.get('applied_steps', 0)) or step
        self._state = None

    def consolidated_state_dict(self):
        """FusedAdamW.state_dict()'s form of the whole state, assembled in rank 0's host memory one tensor at a time
        (the full fp32 state is never held on a GPU); None on the other ranks.  Every rank of the group must call it."""
        if self.world_size > 1 and not self._collective:
            raise RuntimeError('consolidated_state_dict needs the process group of all %d ranks' % self.world_size)
        dist = torch.distributed
        sd = FusedAdamW.state_dict(self)           # param groups with parameter indices, applied_steps, empty state
        sd['applied_steps'] = self._applied_steps()
        if not self._step:                          # nothing stepped yet: FusedAdamW has no state either
            return sd if self.rank == 0 else None
        S, dev = self.shard_size, self.master.device
        for j, (p, o, n) in enumerate(zip(self._params, self.layout['offsets'], self.layout['numels'])):
            if self.rank == 0:
                full = torch.empty((3, n), dtype=torch.float32)
            for q in range(self.world_size):
                a, b = max(o, q * S), min(o + n, (q + 1) * S)
                if a >= b:
                    continue
                if q == self.rank:
                    piece = torch.stack([getattr(self, k)[a - q * S:b - q * S] for k in self._FP32_STATE])
                    if q == 0:
                        full[:, a - o:b - o] = piece.cpu()
                    else:
                        dist.send(piece.contiguous(), dst=self._global_rank(0), group=self.process_group)
                elif self.rank == 0:
                    buf = torch.empty((3, b - a), dtype=torch.float32, device=dev)
                    dist.recv(buf, src=self._global_rank(q), group=self.process_group)
                    full[:, a - o:b - o] = buf.cpu()
            if self.rank == 0:
                sd['state'][j] = {'step': self._step, 'master': full[0].view(p.shape).clone(),
                                  'exp_avg': full[1].view(p.shape).clone(), 'exp_avg_sq': full[2].view(p.shape).clone()}
        return sd if self.rank == 0 else None
