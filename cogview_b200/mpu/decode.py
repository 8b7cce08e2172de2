"""Single-token decode step on the K|V cache.

This is the fast path behind GPT2Model.forward when it is called the way generation/sampling.py:147-151 calls
it (one new token per sequence, `mems` returned by the previous call, mems_mode 'kv').

Two device paths:
  * default: one kernel per operation (cv_linear_small_m, cv_attn_decode, cv_ln_pair_small_m; batch <= 16), CUDA-graph
    captured; in generation runs followed by ONE sampling kernel (cv_sample_topk) inside the same graph.
  * COGVIEW_B200_PERSISTENT=1 and batch <= 8: the whole step — embedding, 48 Sandwich-LN layers, final LayerNorm,
    logits — is ONE persistent kernel (cv_decode_step, csrc/decode_step.cu: bulk-copy weight stream through a
    shared-memory byte ring, register-resident residual stream, grid barriers between the dependency points).  Parity-
    green and profiled per phase (tools/step_prof.py); it is opt-in, the per-operation path is the default.
"""
import os

import torch
import torch.nn.functional as F

from .. import ops
from .layers import _as_bf16


def _persistent_enabled():
    return os.environ.get('COGVIEW_B200_PERSISTENT', '0') == '1'


class DecodeRunner:
    def __init__(self, model, caches, use_graph=True):
        tr = model.transformer
        self.model = model
        self.caches = caches
        self.b = caches.b
        self.heads = tr.num_attention_heads
        self.h = tr.hidden_size
        dev = caches.buf.device
        self.ids = torch.zeros((self.b, 1), dtype=torch.int64, device=dev)
        self.pos = torch.zeros((self.b, 1), dtype=torch.int64, device=dev)
        self.cur_len = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step_logits = None          # output buffer of the step (static: graphs write into it)
        self.graph = None
        self.use_graph = use_graph
        self.persistent = (_persistent_enabled() and self.b <= ops.DECODE_STEP_MAX_BATCH and self.h % 256 == 0
                           and self.h <= 2560)
        # enough (batch, head, split) CTAs to cover the SMs
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        # the key range of every (batch, head) is split so that ~8 CTAs per SM stream the K|V cache: the kernel is
        # latency-bound per CTA, so one CTA per (batch, head) pair alone cannot fill the SMs
        self.nsplit = max(1, min(16, -(-8 * sms // (self.b * self.heads))))
        self.params = None
        self.param_sig = None
        self.graph_launches = 0   # kernels per captured step
        self.replays = 0
        self.last_t = -1
        # token-generation runs (model step + sampling in one graph, next token fed back on the device)
        self.sample_graphs = {}
        self.out_buf = torch.zeros((self.b, caches.maxlen + 1), dtype=torch.int64, device=dev)
        self.stepc = torch.zeros((1, 1), dtype=torch.int64, device=dev)
        self.score_acc = torch.zeros(self.b, dtype=torch.float32, device=dev)
        self.seed_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self.done = torch.zeros(1, dtype=torch.int32, device=dev)
        # sparse inference on the device (is_sparse == 2): text flags of every position, the per-layer key index lists of
        # the current step (cv_sparse_plan) and their common length
        self.sparse = None               # dict(n_img) while a sparse run is being captured / replayed
        self.window = tr.query_window * tr.key_window_times
        self.nmax = tr.num_pivot + self.window
        self.is_txt = None

    # -- parameters --------------------------------------------------------------------------------------------
    def _signature(self):
        """(data_ptr, version) of every parameter the step reads: a load_state_dict / optimizer step / .to() after
        the first generation must not leave the decode path on stale copies or stale pointers."""
        return tuple((p.data_ptr(), p._version) for p in self.model.parameters())

    def _gather_params(self):
        tr = self.model.transformer
        self.params = [tuple(_as_bf16(p.detach()).contiguous() for p in layer.param_list()) for layer in tr.layers]
        self.wte = _as_bf16(self.model.word_embeddings.weight.detach()).contiguous()
        self.wpe = _as_bf16(tr.position_embeddings.weight.detach()).contiguous()
        self.fl = (_as_bf16(tr.final_layernorm.weight.detach()).contiguous(),
                   _as_bf16(tr.final_layernorm.bias.detach()).contiguous(), tr.final_layernorm.eps)
        self.eps = tr.layers[0].layernorm_epsilon
        self.param_sig = self._signature()
        dev = self.ids.device
        if self.persistent:
            table = torch.tensor([[t.data_ptr() for t in P] for P in self.params], dtype=torch.int64)
            self.layer_table = table.to(dev)
            self.workspace = ops.decode_step_workspace(self.h, self.heads, dev)
            self.step_logits = torch.empty((self.b, self.wte.shape[0]), dtype=torch.float32, device=dev)
        # captured graphs hold the old pointers
        self.graph = None
        self.sample_graphs = {}

    def _check_params(self):
        if self.params is None or self.param_sig != self._signature():
            self._gather_params()

    # -- one step ----------------------------------------------------------------------------------------------
    def _ensure_sparse_buffers(self):
        if self.is_txt is None:
            dev = self.ids.device
            L = len(self.model.transformer.layers)
            self.is_txt = torch.zeros((self.b, self.caches.maxlen + 1), dtype=torch.uint8, device=dev)
            self.key_idx = torch.zeros((L, self.b, self.nmax), dtype=torch.int32, device=dev)
            self.n_keys = torch.zeros(1, dtype=torch.int32, device=dev)
            self.plan_err = torch.zeros(1, dtype=torch.int32, device=dev)
            self.len64 = torch.zeros((1, 1), dtype=torch.int64, device=dev)

    def _run(self):
        if self.persistent and self.sparse is None:
            ops.decode_step(self.layer_table, len(self.params), self.heads, self.eps, self.fl[2], self.wte, self.wpe,
                            self.fl[0], self.fl[1], self.ids, self.pos, self.cur_len, self.caches.buf,
                            self.step_logits, self.workspace)
            return self.step_logits
        return self._run_per_op()

    def _run_per_op(self):
        b, h, heads = self.b, self.h, self.heads
        L = len(self.params)
        scal = ops.new_scalars(2 * L + 1, self.ids.device)
        sparse = self.sparse
        if sparse is not None:
            # the fed token's text flag, then the key lists of all layers for this step (pivots are fresh per layer and
            # per token as in mpu/sparse_transformer.py:591-600, drawn on the device)
            tr = self.model.transformer
            self.is_txt.scatter_(1, self.len64.expand(b, 1), (self.ids >= sparse['n_img']).to(torch.uint8))
            ops.sparse_plan(self.is_txt, self.cur_len, L, self.window, tr.num_pivot, tr.max_sequence_length, self.seed_dev,
                            self.key_idx, self.n_keys, self.plan_err)
        x = ops.embed_fwd(self.ids, self.pos, self.wte, self.wpe, scal[2 * L:2 * L + 1])
        prev_gemm = prev_am = prev_post = None
        for i, P in enumerate(self.params):
            (g1, b1, wqkv, bqkv, wd, bd, g3, b3, g2, b2, w1, bb1, w2, bb2, g4, b4) = P
            s = scal[2 * i:2 * i + 2]
            # x_i = x_{i-1} + LN4(mlp_out_{i-1});  xn = LN1(x_i)
            y, xn = ops.ln_pair_small_m(x, prev_gemm, prev_am, prev_post, (g1, b1), self.eps,
                                        want_res_out=prev_gemm is not None)
            if y is not None:
                x = y
            qkv = ops.linear_small_m(xn, wqkv, bqkv)
            if sparse is not None:
                ctx = ops.attn_decode_gather(qkv, self.caches.buf[i], heads, self.cur_len, self.key_idx[i], self.n_keys,
                                             nsplit=self.nsplit)
            else:
                ctx = ops.attn_decode(qkv, self.caches.buf[i], heads, cur_len_dev=self.cur_len, nsplit=self.nsplit)
            attn_out = ops.linear_small_m(ctx, wd, bd, absmax=s[0:1])
            # y = x + LN3(attn_out);  xn2 = LN2(y)
            x, xn2 = ops.ln_pair_small_m(x, attn_out, s[0:1], (g3, b3), (g2, b2), self.eps)
            h4 = ops.linear_small_m(xn2, w1, bb1, act=ops.ACT_GELU)
            prev_gemm = ops.linear_small_m(h4, w2, bb2, absmax=s[1:2])
            prev_am, prev_post = s[1:2], (g4, b4)
        _, xf = ops.ln_pair_small_m(x, prev_gemm, prev_am, prev_post, (self.fl[0], self.fl[1]), self.fl[2],
                                    want_res_out=False)
        if self.step_logits is None:
            self.step_logits = torch.empty((b, self.wte.shape[0]), dtype=torch.float32, device=self.ids.device)
        return ops.linear_small_m(xf, self.wte, out=self.step_logits)

    def step(self, ids, pos, t):
        """ids, pos: [b, 1] int64; t: tokens already cached.  Returns logits [b, V] fp32 (a static buffer that the
        next step overwrites; the sampling graphs never modify it)."""
        if self.params is None or t <= self.last_t:      # a new sequence: make sure the weights are the live ones
            self._check_params()
        self.last_t = t
        self.ids.copy_(ids)
        self.pos.copy_(pos)
        self.cur_len.fill_(t)
        if not self.use_graph:
            self._run()
        elif self.graph is None:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._run()
                self._run()
            torch.cuda.current_stream().wait_stream(side)
            from .._lib import lib
            before = lib().cv_launch_count()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._run()
            self.graph_launches = int(lib().cv_launch_count() - before)
            self.graph.replay()
            self.replays += 1
        else:
            self.graph.replay()
            self.replays += 1
        return self.step_logits

    # -- generation runs: generation/sampling.py:147-183 with nothing left on the host per token -----------------
    def _sample_body(self, key):
        """One token: decode step, then the reference's sampling tail — temperature, invalid vocabulary slices,
        top-k (generation/sampling.py:24-33), softmax, multinomial draw, beam log-probability — and the hand-over of
        the sampled token to the next step, all through device-side state.  With the fused kernel the tail is ONE
        launch (cv_sample_topk, own counter-based generator); COGVIEW_B200_FUSED_SAMPLING=0 keeps the reference's
        torch operations (torch.multinomial's generator) instead."""
        temperature, top_k, inv = key[:3]
        logits = self._run()
        if self.sparse is not None:
            self.len64.add_(1)
        vocab = logits.shape[1]
        valid = ops.valid_ranges(inv, vocab)
        if os.environ.get('COGVIEW_B200_FUSED_SAMPLING', '1') != '0' and 1 <= len(valid) <= 4:
            ops.sample_topk(logits, temperature, top_k, valid, seed_dev=self.seed_dev, step=self.stepc,
                            next_ids=self.ids, out_tokens=self.out_buf, score_acc=self.score_acc, pos=self.pos,
                            cur_len=self.cur_len, done=self.done)
            return
        logits = logits.clone()
        logits.div_(temperature)
        for a, z in inv:
            logits[:, a:z] = -float('Inf')
        if top_k > 0:
            kth = torch.topk(logits, top_k)[0][..., -1, None]
            logits.masked_fill_(logits < kth, -float('Inf'))
        probs = F.softmax(logits, dim=-1)
        prev = torch.multinomial(probs, num_samples=1)
        self.score_acc.add_(torch.log(torch.gather(probs, 1, prev)[:, 0]))
        self.out_buf.scatter_(1, self.stepc.expand(self.b, 1), prev)
        self.stepc.add_(1)
        self.ids.copy_(prev)
        self.pos.add_(1)
        self.cur_len.add_(1)

    def _reset_run(self, ids, pos, t):
        self.ids.copy_(ids)
        self.pos.copy_(pos)
        self.cur_len.fill_(t)
        self.stepc.zero_()
        self.score_acc.zero_()
        if self.sparse is not None:      # text flags of the history, flag cursor (the warm-up steps before a capture moved them)
            flags = self.sparse['flags']
            self.is_txt.zero_()
            self.is_txt[:, :flags.shape[1]] = flags
            self.len64.fill_(t)
            self.plan_err.zero_()

    def sample_run(self, ids, pos, t, n_steps, temperature, top_k, invalid_slices, sparse=None):
        """n_steps tokens starting from `ids` ([b, 1], at positions `pos`, t tokens cached).  One graph replay per
        token.  Returns (tokens [b, n_steps] int64, summed log-probabilities [b] fp32).
        sparse: None, or dict(n_img=..., tokens=[b, t + 1] every token so far) for is_sparse == 2."""
        self._check_params()
        self.last_t = t + n_steps
        vocab = self.model.word_embeddings.weight.shape[0]
        key = (float(temperature), int(top_k), tuple(sl.indices(vocab)[:2] for sl in invalid_slices),
               None if sparse is None else int(sparse['n_img']))
        assert n_steps <= self.out_buf.shape[1]
        self.sparse = None
        if sparse is not None:
            self._ensure_sparse_buffers()
            hist = sparse['tokens']
            assert hist.shape == (self.b, t + 1)
            self.sparse = dict(n_img=int(sparse['n_img']), flags=(hist >= int(sparse['n_img'])).to(torch.uint8))
        self._reset_run(ids, pos, t)
        # the draw generator of the fused tail: a fresh seed per run from torch's (seedable) host generator
        self.seed_dev.copy_(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64), non_blocking=True)
        graph = self.sample_graphs.get(key)
        if graph is None and self.use_graph:
            dev = self.ids.device
            rng = torch.cuda.get_rng_state(dev)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):           # warm-up (allocator, lazy init); its side effects are undone below
                self._sample_body(key)
                self._sample_body(key)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.set_rng_state(rng, dev)
            self._reset_run(ids, pos, t)
            from .._lib import lib
            before = lib().cv_launch_count()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._sample_body(key)
            self.graph_launches = int(lib().cv_launch_count() - before)   # this library's kernels per replayed token
            self.sample_graphs[key] = graph
        for _ in range(n_steps):
            if graph is None:
                self._sample_body(key)
            else:
                graph.replay()
        self.replays += n_steps
        if self.sparse is not None:
            self.sparse = None
            if int(self.plan_err.item()) != 0:
                raise RuntimeError('sparse decode: the key list did not fit num_pivot + window entries')
        return self.out_buf[:, :n_steps].clone(), self.score_acc.clone()
