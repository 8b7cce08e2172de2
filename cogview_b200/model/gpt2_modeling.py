"""GPT-2 model — mirror of the reference's model/gpt2_modeling.py (GPT2Model :55-123,
gpt2_get_params_for_weight_decay_optimization :35-52): same constructor and forward signatures, same
state_dict keys (`word_embeddings.weight`, `transformer.*`)."""
import os

import torch

from .. import mpu, ops
from ..mpu.layers import _as_bf16
from ..mpu.sparse_transformer import _EmbedFn, mask_to_sep


def init_method_normal(std=0.02):
    def init_(tensor):
        return torch.nn.init.normal_(tensor, mean=0.0, std=std)
    return init_


def gpt2_get_params_for_weight_decay_optimization(module):
    """Weights decay; biases and LayerNorm parameters do not (model/gpt2_modeling.py:35-52)."""
    weight_decay_params = {'params': []}
    no_weight_decay_params = {'params': [], 'weight_decay': 0.0}
    for module_ in module.modules():
        if isinstance(module_, (mpu.LayerNorm, torch.nn.LayerNorm)):
            no_weight_decay_params['params'].extend([p for p in list(module_._parameters.values()) if p is not None])
        else:
            weight_decay_params['params'].extend(
                [p for n, p in list(module_._parameters.items()) if p is not None and n != 'bias'])
            no_weight_decay_params['params'].extend(
                [p for n, p in list(module_._parameters.items()) if p is not None and n == 'bias'])
    return weight_decay_params, no_weight_decay_params


class _LogitsFn(torch.autograd.Function):
    """logits = h W^T with the tied word-embedding matrix (model/gpt2_modeling.py:117-118), fp32 output."""

    @staticmethod
    def forward(ctx, hidden, weight):
        w = _as_bf16(weight)
        ctx.save_for_backward(hidden, w)
        ctx.wdtype = weight.dtype
        V = w.shape[0]
        ld = (V + 3) // 4 * 4
        out = torch.empty((hidden.shape[0], ld), dtype=torch.float32, device=hidden.device)
        ops.gemm(hidden, w, out_dtype=torch.float32, out=out[:, :V] if ld != V else out)
        return out[:, :V]

    @staticmethod
    def backward(ctx, d_logits):
        hidden, w = ctx.saved_tensors
        dl = _as_bf16(d_logits)
        if dl.stride(1) != 1 or dl.stride(0) % 8 != 0:
            V = dl.shape[1]
            buf = torch.empty((dl.shape[0], (V + 7) // 8 * 8), dtype=torch.bfloat16, device=dl.device)
            buf[:, :V].copy_(dl)
            dl = buf[:, :V]
        d_hidden = ops.gemm(dl, w, b_mn_major=True)
        d_w = ops.gemm(dl, hidden, a_mn_major=True, b_mn_major=True)
        return d_hidden, d_w.to(ctx.wdtype)


class _VocabXentFn(torch.autograd.Function):
    """Per-token loss = logsumexp(h W^T) - (h W^T)[target] with the tied word-embedding matrix, without the fp32
    logits: the values vocab_parallel_cross_entropy(_LogitsFn(h, W), target) gives, from the same fp32 GEMM
    accumulators (only the order of the sum of exponentials differs).  The forward keeps h, the bf16 weight, the
    targets and the row log-sum-exp; the backward recomputes the logits one vocabulary chunk at a time
    (ops.vocab_xent_bwd: bf16 dlogits as in the logits route, dH summed over chunks in fp32 when there are several,
    dW written per chunk) and never holds an [M, V] tensor.  Repeats with equal inputs and budget are bit-equal."""

    @staticmethod
    def forward(ctx, hidden, weight, target, chunk_bytes):
        w = _as_bf16(weight)
        loss, lse = ops.vocab_xent_fwd(hidden, w, target)
        ctx.save_for_backward(hidden, w, target, lse)
        ctx.wdtype = weight.dtype
        ctx.chunk_bytes = chunk_bytes
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        hidden, w, target, lse = ctx.saved_tensors
        d_hidden, d_w = ops.vocab_xent_bwd(hidden, w, target, lse, grad_loss, ctx.chunk_bytes)
        return d_hidden, d_w.to(ctx.wdtype), None, None


class GPT2Model(torch.nn.Module):
    """GPT-2 language model over concatenated text + image tokens.  forward returns (logits, *mems)."""

    def __init__(self, num_layers, vocab_size, hidden_size, num_attention_heads, embedding_dropout_prob,
                 attention_dropout_prob, output_dropout_prob, max_sequence_length, max_memory_length,
                 checkpoint_activations, checkpoint_num_layers=1, parallel_output=True, query_window=128,
                 key_window_times=6, num_pivot=768):
        super().__init__()
        self.parallel_output = parallel_output
        init_method = init_method_normal(std=0.02)
        self.word_embeddings = mpu.VocabParallelEmbedding(vocab_size, hidden_size, init_method=init_method)
        self.transformer = mpu.GPT2ParallelTransformer(
            num_layers, hidden_size, num_attention_heads, max_sequence_length, max_memory_length,
            embedding_dropout_prob, attention_dropout_prob, output_dropout_prob, checkpoint_activations,
            checkpoint_num_layers, query_window=query_window, key_window_times=key_window_times, num_pivot=num_pivot)

    def forward(self, input_ids, position_ids, attention_mask, txt_indices_bool, img_indices_bool, is_sparse, *mems,
                logits_last_only=False, labels=None, xent_chunk_bytes=None):
        """Same positional arguments as the reference (model/gpt2_modeling.py:106).  Returns
        (logits [b, s, V] fp32, *mems).  `logits_last_only` (keyword, extension): only the last position's
        logits are computed — what the sampling loop reads (generation/sampling.py:155).
        `labels` (keyword, extension; int64 [b, s]): returns (losses [b, s] fp32, *mems) instead, the per-token
        loss vocab_parallel_cross_entropy(logits.float(), labels) gives, computed without the logits
        (_VocabXentFn; with and without autograd, never on the decode fast path).  The backward's dlogits chunk
        budget is `xent_chunk_bytes` (default ops.XENT_CHUNK_BYTES).  A label outside [0, V) gives a NaN loss."""
        if labels is not None and logits_last_only:
            raise ValueError('labels= and logits_last_only=True cannot be combined: the loss needs every position')
        tr = self.transformer
        b, sq = input_ids.shape
        if labels is not None and tuple(labels.shape) != (b, sq):
            raise ValueError('labels must have the shape of input_ids %s, got %s' % ((b, sq), tuple(labels.shape)))
        mem_len = mems[0].size(1) if mems else 0
        sep = 0 if is_sparse != 0 else mask_to_sep(attention_mask, sq, sq + mem_len)
        if position_ids.shape != input_ids.shape:
            position_ids = position_ids.expand_as(input_ids)
        fast = self._fast_decode(input_ids, position_ids, mems, b, sq) if is_sparse == 0 and labels is None else None
        if fast is not None:
            return fast
        wte, wpe = self.word_embeddings.weight, tr.position_embeddings.weight
        if torch.is_grad_enabled() and (wte.requires_grad or wpe.requires_grad):
            p_emb = tr.embedding_dropout_prob if tr.training else 0.0
            x, am_x = _EmbedFn.apply(input_ids, position_ids, wte, wpe, p_emb)
        else:
            am_x = ops.new_scalars(1, wte.device)
            x = ops.embed_fwd(input_ids, position_ids, _as_bf16(wte.detach()).contiguous(),
                              _as_bf16(wpe.detach()).contiguous(), am_x)
        y, mem_layers = tr.run_layers(x, am_x, b, sq, sep, mems, is_sparse=is_sparse,
                                      txt_indices_bool=txt_indices_bool, img_indices_bool=img_indices_bool)
        if labels is not None:
            target = labels.reshape(-1).to(device=y.device, dtype=torch.long)
            if torch.is_grad_enabled() and (y.requires_grad or wte.requires_grad):
                losses = _VocabXentFn.apply(y, wte, target, xent_chunk_bytes)
            else:
                losses, _ = ops.vocab_xent_fwd(y, _as_bf16(wte.detach()), target)
            return (losses.view(b, sq), *mem_layers)
        h = y.shape[1]
        if logits_last_only:
            y = y.view(b, sq, h)[:, -1].contiguous()
            sq_out = 1
        else:
            sq_out = sq
        if torch.is_grad_enabled() and (y.requires_grad or wte.requires_grad):
            logits = _LogitsFn.apply(y, wte)
        else:
            logits = _LogitsFn.forward(_NoCtx(), y, wte.detach())
        return (logits.view(b, sq_out, -1), *mem_layers)


def _fast_decode_impl(self, input_ids, position_ids, mems, b, sq):
    """One token per sequence on the K|V cache (the call pattern of generation/sampling.py:147-151): CUDA-graph
    replay of the weight-streaming decode step.  Returns None when the call does not qualify."""
    tr = self.transformer
    if (sq != 1 or not mems or tr.mems_mode != 'kv' or tr.max_memory_length <= 0 or torch.is_grad_enabled()
            or not ops.decode_batch_supported(b, tr.hidden_size)
            or os.environ.get('COGVIEW_B200_FAST_DECODE', '1') == '0'):
        return None
    from ..mpu import kv_cache
    from ..mpu.decode import DecodeRunner
    caches = kv_cache.prepare(tr, mems, b, sq)
    runner = getattr(caches, 'runner', None)
    if runner is None:
        runner = caches.runner = DecodeRunner(self, caches,
                                              use_graph=os.environ.get('COGVIEW_B200_CUDA_GRAPH', '1') != '0')
    logits = runner.step(input_ids, position_ids, caches.t)
    return (logits.view(b, 1, -1), *caches.views())


GPT2Model._fast_decode = _fast_decode_impl


def _generate_run_impl(self, last_tokens, first_pos, mems, n_steps, temperature, top_k, invalid_slices, sparse=None,
                       row_pad=None, top_p=0.0, forced=None):
    """n_steps sampled tokens in a row on the K|V cache — the inner loop of generation/sampling.py:147-183 for a
    stretch of the template that is all 'generate' slots — with the sampling tail inside the replayed CUDA graph
    (mpu/decode.py sample_run).  Returns None when the fast path does not apply, else
    (tokens [b, n_steps], summed log-probabilities [b], mems).
    sparse = dict(n_img=<image vocabulary size>, tokens=<[b, t + 1] all tokens so far>) runs the stretch with
    is_sparse == 2 semantics (mpu/sparse_transformer.py:498-520, :591-600, :727-750): pivots + trailing window per layer per
    token, chosen on the device (cv_sparse_plan) instead of Python's random.sample — same distribution, other stream.
    first_pos is one position for every row, or one per row (a sequence or 1-D tensor of b positions).
    row_pad (int32 [b] on the device, from mpu/kv_cache.py assemble): row i of `mems` holds mems[0].size(1) - row_pad[i]
    tokens — rows of prompts of different lengths in one run (not with sparse).
    top_p > 0 adds nucleus filtering after top-k (generation/sampling.py:34-47) to the sampling tail.
    forced (int64 [b, n_steps] or None; not with sparse): where forced[i, j] >= 0, that given token replaces row i's
    draw at step j, in the returned tokens and as the input of step j + 1 (generation.sampling.filling_completions:
    given codes inside a completed region).  The log-probabilities of such rows include the replaced draws and mean
    nothing."""
    tr = self.transformer
    b = last_tokens.shape[0]
    if (not mems or tr.mems_mode != 'kv' or tr.max_memory_length <= 0 or torch.is_grad_enabled()
            or not ops.decode_batch_supported(b, tr.hidden_size) or n_steps < 1
            or os.environ.get('COGVIEW_B200_FAST_DECODE', '1') == '0'
            or os.environ.get('COGVIEW_B200_GRAPH_SAMPLING', '1') == '0'):
        return None
    from ..mpu import kv_cache
    from ..mpu.decode import DecodeRunner
    if mems[0].size(1) + n_steps > tr.max_memory_length:
        return None
    caches = kv_cache.prepare(tr, mems, b, n_steps)
    runner = getattr(caches, 'runner', None)
    if runner is None:
        runner = caches.runner = DecodeRunner(self, caches,
                                              use_graph=os.environ.get('COGVIEW_B200_CUDA_GRAPH', '1') != '0')
    if torch.is_tensor(first_pos) or isinstance(first_pos, (list, tuple)):
        pos = torch.as_tensor(first_pos, dtype=torch.long).to(last_tokens.device).reshape(b, 1)
    else:
        pos = torch.full((b, 1), int(first_pos), dtype=torch.long, device=last_tokens.device)
    # sparse inference: cv_sparse_plan is written for at most 16 sequences
    if sparse is not None and (b > ops.DECODE_SMALL_MAX_BATCH or tr.max_memory_length > 4096 or row_pad is not None
                               or forced is not None):
        return None
    new_tokens, logp = runner.sample_run(last_tokens.reshape(b, 1), pos, caches.t, n_steps, temperature, top_k,
                                         invalid_slices, sparse=sparse, row_pad=row_pad, top_p=top_p, forced=forced)
    return new_tokens, logp, caches.views()


GPT2Model.generate_run = _generate_run_impl


def _shared_run_impl(self, last_tokens, first_pos, mems, n_steps, temperature, top_k, invalid_slices):
    """generate_run for rows that share prompts: `mems` are the K|V-cache views GPT2Model.forward returned for
    `groups` prompts of one length P (the pooled cache of batch size groups), and the b rows of last_tokens [b, 1]
    (b a multiple of groups) are their beams, G = b / groups consecutive rows per prompt, all at position first_pos.
    Each prompt's K|V stays once in that cache and is read by cv_attn_decode_shared for all of its beams
    (DecodeRunner's shared mode); the rows' own tokens go to a suffix cache of n_steps slots (kv_cache.shared).
    Returns None when the fast path does not apply, else (tokens [b, n_steps], summed log-probabilities [b])."""
    tr = self.transformer
    b = last_tokens.shape[0]
    if (not mems or tr.mems_mode != 'kv' or tr.max_memory_length <= 0 or torch.is_grad_enabled()
            or not ops.decode_batch_supported(b, tr.hidden_size) or n_steps < 1
            or os.environ.get('COGVIEW_B200_FAST_DECODE', '1') == '0'
            or os.environ.get('COGVIEW_B200_GRAPH_SAMPLING', '1') == '0'):
        return None
    from ..mpu import kv_cache
    from ..mpu.decode import DecodeRunner
    groups, P = mems[0].size(0), mems[0].size(1)
    prefix = tr.__dict__.get('_kv_pool', {}).get(groups)
    if b % groups != 0 or b // groups > 64 or P < 1 or prefix is None or not prefix.matches(mems, groups):
        return None
    caches = kv_cache.shared(tr, prefix, P, b, n_steps)
    try:
        runner = caches.runner
        if runner is None:
            runner = caches.runner = DecodeRunner(self, caches,
                                                  use_graph=os.environ.get('COGVIEW_B200_CUDA_GRAPH', '1') != '0')
        pos = torch.full((b, 1), int(first_pos), dtype=torch.long, device=last_tokens.device)
        return runner.sample_run(last_tokens.reshape(b, 1), pos, 0, n_steps, temperature, top_k, invalid_slices)
    finally:
        caches.prefix = None


GPT2Model.shared_run = _shared_run_impl


def _chunk_run_impl(self, tokens, position_ids, mems, row_pad=None):
    """n given tokens per row on the K|V cache in one eager pass — the model call generation/sampling.py:147-151
    makes for a template stretch of provided tokens (plus the last sampled one), for a batch whose rows sit at
    different cache lengths.  tokens, position_ids: int64 [b, n] (positions per row: every row has its own [ROI2]
    offset); mems: the pooled cache views of kv_cache.assemble or of a previous generate_run / chunk_run; row_pad:
    int32 [b] on the device or None, row i holding mems[0].size(1) - row_pad[i] tokens.  The attention of every layer
    is cv_attn_chunk_ragged (each row against its own prefix, the chunk's K|V appended at the row's own length); the
    linears and LayerNorms are the general kernels over the b*n rows, and the abs-max LayerNorm scales are taken over
    the whole batch — so a row matches the same tokens run alone through forward within bf16 tolerance, not bit for
    bit.  Returns (last position's logits [b, V] fp32, mems): every row's length grows by n, row_pad is unchanged, so
    a following generate_run(..., row_pad=row_pad) continues each row at its own length.  None when the call does
    not qualify (no K|V-cache mems, autograd on, n outside 1..ops.ATTN_CHUNK_MAX, or cache overflow)."""
    tr = self.transformer
    b, n = tokens.shape
    if (not mems or tr.mems_mode != 'kv' or tr.max_memory_length <= 0 or torch.is_grad_enabled()
            or not 1 <= n <= ops.ATTN_CHUNK_MAX or mems[0].size(1) + n > tr.max_memory_length
            or position_ids.shape != tokens.shape or mems[0].size(0) != b):
        return None
    t = mems[0].size(1)
    heads = tr.num_attention_heads
    nsplit = ops.attn_chunk_nsplit(b, heads, t + n, tokens.device)
    work = None
    if nsplit > 1:
        work = torch.empty(ops.lib().cv_attn_chunk_workspace_bytes(b, heads, n, nsplit) // 4, dtype=torch.float32,
                           device=tokens.device)

    def chunk_attn(i, caches):
        cache_i = caches.buf[i]

        def attn(q):
            # q is the first third of the packed QKV GEMM output [b, n, 3h]: the kernel reads q | k | v in place
            qkv = q.as_strided((b, n, q.shape[2] * 3), (q.stride(0), q.stride(1), 1))
            return ops.attn_chunk_ragged(qkv, cache_i, heads, t, row_pad, nsplit=nsplit, workspace=work)
        return attn

    wte, wpe = self.word_embeddings.weight, tr.position_embeddings.weight
    am_x = ops.new_scalars(1, wte.device)
    x = ops.embed_fwd(tokens, position_ids, _as_bf16(wte.detach()).contiguous(), _as_bf16(wpe.detach()).contiguous(),
                      am_x)
    y, mem_layers = tr.run_layers(x, am_x, b, n, 0, mems, chunk_attn=chunk_attn)
    y = y.view(b, n, -1)[:, -1].contiguous()
    logits = _LogitsFn.forward(_NoCtx(), y, wte.detach())
    return logits, mem_layers


GPT2Model.chunk_run = _chunk_run_impl


def _token_logprobs_impl(self, input_ids, position_ids, attention_mask, score_index, targets, vocab_begin=0,
                         vocab_end=None, *, is_sparse=0):
    """log_softmax over the vocabulary window [vocab_begin, vocab_end) of the logits at a few positions, picked at
    their targets: what generation/sampling.py:214-230 reads of a full forward, without the forward's logits or
    memory.  input_ids, position_ids int64 [b, s]; attention_mask as forward takes it; score_index int64 flat
    indices into the b*s rows; targets int64 [len(score_index)] (a target outside the window gives -inf).  Returns
    fp32 [len(score_index)].  The layers run with no memory kept (run_layers(keep_mems=False): no K|V cache is
    prepared and the pooled caches stay as they are); only the scored rows of the bf16 final-LN output go through
    cv_vocab_logprob, which never writes a logit to memory.  torch.no_grad() and dense attention (is_sparse=0) only."""
    if torch.is_grad_enabled():
        raise RuntimeError('token_logprobs runs under torch.no_grad() only')
    if is_sparse != 0:
        raise NotImplementedError('token_logprobs supports dense attention (is_sparse=0) only')
    tr = self.transformer
    b, sq = input_ids.shape
    sep = mask_to_sep(attention_mask, sq, sq)
    if position_ids.shape != input_ids.shape:
        position_ids = position_ids.expand_as(input_ids)
    wte, wpe = self.word_embeddings.weight, tr.position_embeddings.weight
    w = _as_bf16(wte.detach()).contiguous()
    am_x = ops.new_scalars(1, wte.device)
    x = ops.embed_fwd(input_ids, position_ids, w, _as_bf16(wpe.detach()).contiguous(), am_x)
    y, _ = tr.run_layers(x, am_x, b, sq, sep, [], keep_mems=False)
    rows = y.index_select(0, score_index.to(device=y.device, dtype=torch.long).view(-1))
    return ops.vocab_logprob(rows, w, targets.to(device=y.device, dtype=torch.long), vocab_begin, vocab_end)


GPT2Model.token_logprobs = _token_logprobs_impl


class _NoCtx:
    def save_for_backward(self, *a):
        pass
