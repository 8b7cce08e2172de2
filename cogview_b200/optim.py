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


class FusedAdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_grad_norm=0.0):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.max_grad_norm = float(max_grad_norm)
        self._scal = None
        self._tables = None          # (pinned host staging x2, device table), rebuilt when the parameter list changes
        self._copied = [None, None]  # CUDA event recorded after the async copy out of each staging buffer
        self._flip = 0
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
        self._tables = None

    _ENTRY = np.dtype([('param', '<u8'), ('grad', '<u8'), ('master', '<u8'), ('m', '<u8'), ('v', '<u8'), ('n', '<i8'),
                       ('lr', '<f4'), ('wd', '<f4'), ('bc1', '<f4'), ('bc2', '<f4')])   # = cv_adamw_entry, 64 bytes

    def _table(self, plist, dev):
        """Fills the device-resident cv_adamw_entry table for this step (gradient pointers may move between steps)."""
        n = len(plist)
        if self._tables is None or self._tables[2].numel() != n * 64 or self._tables[2].device != dev:
            host = [torch.empty(n * 64, dtype=torch.uint8).pin_memory() for _ in range(2)]
            self._tables = (host[0], host[1], torch.empty(n * 64, dtype=torch.uint8, device=dev))
            self._copied = [None, None]
        self._flip ^= 1                                   # double-buffered: the previous step's copy may be in flight
        if self._copied[self._flip] is not None:          # the copy issued two steps ago has long finished; make sure
            self._copied[self._flip].synchronize()
        host = self._tables[self._flip]
        rec = host.numpy().view(self._ENTRY)
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
        self._tables[2].copy_(host, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._copied[self._flip] = ev
        return self._tables[2]

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
        L = lib()
        stream = stream_ptr()
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
            if self._scal is None or self._scal.device != dev:
                self._scal = torch.zeros(3, dtype=torch.float32, device=dev)
            if self._state is None or self._state.device != dev:
                self._state = torch.tensor([0, self._applied], dtype=torch.int32, device=dev)
            self._scal.zero_()
            check(L.cv_sumsq_bf16_multi(ptr(table), len(plist), ptr(self._scal[0:1]), stream), "cv_sumsq_bf16_multi")
            check(L.cv_clip_coef(ptr(self._scal[0:1]), self.max_grad_norm, ptr(self._scal[1:2]), ptr(self._scal[2:3]),
                                 ptr(self._state), stream), "cv_clip_coef")
            coef = self._scal[1:2]
            self.last_grad_norm = self._scal[2:3]
        check(L.cv_adamw_step_multi(ptr(table), len(plist), float(b1), float(b2), float(eps), ptr(coef), 1.0,
                                    ptr(self._state) if self.max_grad_norm > 0 else 0, stream), "cv_adamw_step_multi")
        return None
