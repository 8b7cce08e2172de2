"""Autoregressive token filling — mirror of the reference's generation/sampling.py (`top_k_logits` :24-49,
`get_batch` :51-63, `filling_sequence` :64-186, `shrink_beams` :188-198, `add_interlacing_beam_marks`
:200-211, `inverse_prompt_score` :214-230) and of `get_masks_and_position_ids` (pretrain_gpt2.py:210-253).

Same call signatures and semantics; two host-side differences that do not change results:
  * the template `seq` is read once into a Python list (the reference indexes a CUDA tensor every step, which
    forces a device sync per generated token);
  * the tokenizer is any object with the UnifiedTokenizer surface the loop uses (`tok['[BOI1]']`,
    `tok.img_tokenizer.num_tokens`, `tok.txt_tokenizer.num_tokens`); `TokenLayout` provides that surface from
    the vocabulary sizes alone (the role FakeTokenizer plays in data_utils/unified_tokenizer.py:208-212).
"""
import math
import os as _os

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------------
# token layout (data_utils/unified_tokenizer.py:23-67): [image codes | text pieces | 27 command tokens]
# ----------------------------------------------------------------------------------------------------
class _Count:
    def __init__(self, n):
        self.num_tokens = n

    def __len__(self):
        return self.num_tokens


class TokenLayout:
    RAW_COMMAND_TOKENS = ['[PAD]', '[BOI1]', '[BOI2]', '[BOI3]', '[EOI1]', '[EOI2]', '[EOI3]', '[ROI1]', '[ROI2]',
                          '[ROI3]', '[SEP]', '[MASK]', '[CLS]', '[ENC]', '[TINY]', '[SMALL]', '[BASE]', '[BIG]',
                          '[POS0]', '[POS1]', '[POS2]', '[POS3]', '[POS4]', '[POS5]', '[POS6]', '[POS7]', '[POS8]']

    def __init__(self, img_tokens=8192, txt_tokens=50000):
        self.img_tokenizer = _Count(img_tokens)
        self.txt_tokenizer = _Count(txt_tokens)
        base = img_tokens + txt_tokens
        self.command_tokens = {k: base + i for i, k in enumerate(self.RAW_COMMAND_TOKENS)}
        self.num_tokens = base + len(self.RAW_COMMAND_TOKENS)

    def __getitem__(self, command_token):
        return self.command_tokens[command_token]

    def wrap_code(self, code, idx=1):
        """data_utils/unified_tokenizer.py:125-151: [size tag] [BOIidx] code [EOIidx]; the tag follows the side of
        the (square) code grid.  Lists, numpy arrays and tensors keep their type."""
        n = len(code)
        side = int(math.sqrt(n) + 1e-4)
        assert side * side == n, 'image codes must form a square grid'
        prefix = {8: '[TINY]', 16: '[SMALL]', 32: '[BASE]', 64: '[BIG]'}[side]
        head = [self.command_tokens[prefix], self.command_tokens['[BOI%d]' % idx]]
        tail = [self.command_tokens['[EOI%d]' % idx]]
        if isinstance(code, list):
            return head + code + tail
        if isinstance(code, np.ndarray):
            return np.concatenate((np.array(head), code, np.array(tail)), axis=0)
        if isinstance(code, torch.Tensor):
            return torch.cat((torch.tensor(head, dtype=code.dtype, device=code.device), code,
                              torch.tensor(tail, dtype=code.dtype, device=code.device)))
        raise ValueError('code must be a list, numpy array or tensor')

    def __len__(self):
        return self.num_tokens


_TOKENIZER = None


def set_tokenizer(tok):
    global _TOKENIZER
    _TOKENIZER = tok


def get_tokenizer(args=None):
    global _TOKENIZER
    if _TOKENIZER is None:
        n_img = getattr(args, 'img_tokenizer_num_tokens', None) or 8192
        _TOKENIZER = TokenLayout(img_tokens=n_img)
    return _TOKENIZER


# ----------------------------------------------------------------------------------------------------
def get_masks_and_position_ids(data, loss_mask=None, attention_mask=None, args=None):
    """pretrain_gpt2.py:210-253: lower-triangular [1,1,s,s] mask, ones loss mask, arange position ids.

    With `args.finetune` and args.max_position_embeddings < args.max_position_embeddings_finetune (the finetune
    branch, :228-247: two-image rows longer than the position table), each row's positions restart at 0 at its
    first [ROI2], which takes position 0 itself, and every position >= max_position_embeddings is then clamped to
    max_position_embeddings - 1.  Computed on the device in one pass (the reference loops over the rows in Python);
    a row without [ROI2] raises AssertionError('Some samples do not have [ROI2]!'), which reads one flag to the host.
    Sampling (filling_sequence) gives the tokens after [ROI2] the same positions 1, 2, ... but keeps [ROI2] itself at
    its own index; that mismatch is the reference's, and this branch keeps its training positions."""
    batch_size, seq_length = data.size()
    if attention_mask is None:
        attention_mask = torch.tril(torch.ones((1, seq_length, seq_length), device=data.device)).unsqueeze(1)
    if loss_mask is None:
        loss_mask = torch.ones(data.size(), dtype=torch.float, device=data.device)
    if (args is not None and getattr(args, 'finetune', False)
            and args.max_position_embeddings < args.max_position_embeddings_finetune):
        ar = torch.arange(seq_length, dtype=torch.long, device=data.device).unsqueeze(0)
        first = torch.where(data == get_tokenizer()['[ROI2]'], ar, seq_length).amin(dim=1, keepdim=True)
        assert bool((first < seq_length).all()), 'Some samples do not have [ROI2]!'
        position_ids = torch.where(ar < first, ar, ar - first).clamp_max(args.max_position_embeddings - 1)
    else:
        position_ids = torch.arange(seq_length, dtype=torch.long, device=data.device).unsqueeze(0).expand_as(data)
    return attention_mask, loss_mask, position_ids


def top_p_logits(logits, top_p, filter_value=-float('Inf')):
    """The nucleus (top-p) filter of top_k_logits (generation/sampling.py:34-47) row by row on [b, V] logits, in
    place: sort each row descending, take the cumulative softmax, shift it by one, and set every logit whose mass
    before it in that order exceeds top_p to filter_value.  Sort, cumsum, a shift and a scatter only, no boolean
    indexing, so it can be captured in a CUDA graph.  Each row gets what the reference's one-row branch gives it."""
    sorted_logits, sorted_indices = torch.sort(logits, descending=True)
    cumulative_probs = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
    remove = cumulative_probs > top_p
    remove[..., 1:] = remove[..., :-1].clone()
    remove[..., 0] = False
    return logits.masked_fill_(torch.zeros_like(remove).scatter_(-1, sorted_indices, remove), filter_value)


def top_k_logits(logits, top_k=0, top_p=0.0, filter_value=-float('Inf')):
    """generation/sampling.py:24-49.  The reference's top-p branch views the logits as one row; logits with more
    than one row go through top_p_logits, which applies it to each row."""
    if top_k > 0:
        kth = torch.topk(logits, top_k)[0][..., -1, None]
        logits[logits < kth] = filter_value
    if top_p > 0.0 and logits.dim() == 2 and logits.shape[0] > 1:
        return top_p_logits(logits, top_p, filter_value)
    if top_p > 0.0:
        logits = logits.view(logits.size()[1]).contiguous()
        sorted_logits, sorted_indices = torch.sort(logits, descending=True)
        cumulative_probs = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
        remove = cumulative_probs > top_p
        remove[..., 1:] = remove[..., :-1].clone()
        remove[..., 0] = 0
        logits[sorted_indices[remove]] = filter_value
        logits = logits.view(1, -1).contiguous()
    return logits


def get_batch(context_tokens, device, args):
    tokens = context_tokens
    tokens = tokens.unsqueeze(0).contiguous() if tokens.dim() == 1 else tokens.view(tokens.shape[0], -1).contiguous()
    tokens = tokens.to(device)
    attention_mask, loss_mask, position_ids = get_masks_and_position_ids(tokens)
    return tokens, attention_mask, position_ids


def shrink_beams(tokens, mems, nb, score):
    """generation/sampling.py:188-198 — keep the best-scoring beam when the beam count shrinks."""
    if tokens.shape[0] == nb:
        return tokens, mems, score
    if torch.is_tensor(score):      # accumulated on the device (no per-token sync); read it only when needed
        score = score.tolist()
    max_idx = score.index(max(score))
    tokens = tokens[max_idx].unsqueeze(0)
    return tokens, [mem[max_idx: max_idx + 1] for mem in mems], [0]


def add_interlacing_beam_marks(seq, nb=12, period=3000):
    """generation/sampling.py:200-211 — replace each -1 (to be generated) by -nb."""
    assert isinstance(seq, list) or len(seq.shape) == 1
    blk_cnt = 0
    for i in range(len(seq)):
        if seq[i] == -1:
            blk_cnt += 1
            seq[i] = -nb
            if blk_cnt == period:
                nb += (nb % 2) * 2 - 1
                blk_cnt = 0
        else:
            blk_cnt = 0


def _slices_after(tokenizer, tok, cur):
    """The vocabulary slices that may not be sampled after token `tok` ([BOI*]: only image codes, [EOI*]: only text)."""
    n_img = tokenizer.img_tokenizer.num_tokens
    n_txt = tokenizer.txt_tokenizer.num_tokens
    if tok in (tokenizer['[BOI1]'], tokenizer['[BOI2]']):
        return [slice(n_img, None)]
    if tok in (tokenizer['[EOI1]'], tokenizer['[EOI2]']):
        return [slice(0, n_img), slice(n_img + n_txt, None)]
    return cur


def _scan_context(tmpl, tokenizer):
    """(context length, position offset of the last [ROI2] in the context or 100000, invalid slices after the
    context) of a template list."""
    offset = 100000
    invalid_slices = [slice(0, tokenizer.img_tokenizer.num_tokens)]
    context_length = 0
    while context_length < len(tmpl) and tmpl[context_length] >= 0:
        invalid_slices = _slices_after(tokenizer, tmpl[context_length], invalid_slices)
        if tmpl[context_length] == tokenizer['[ROI2]']:
            offset = context_length
        context_length += 1
    return context_length, offset, invalid_slices


def _next_token_probs(logits, invalid_slices, args):
    """Sampling distribution [b, V] from the last position's logits [b, s, V] (modified in place)."""
    logits = logits[:, -1]
    logits /= args.temperature
    for sl in invalid_slices:
        logits[..., sl] = -float('Inf')
    logits = top_k_logits(logits, top_k=args.top_k, top_p=args.top_p)
    return F.softmax(logits, dim=-1)


def filling_sequence(model, seq, args, mems=None, invalid_slices=[], **kwargs):
    """generation/sampling.py:64-186.  seq: 1-D LongTensor template [ctx..., -N (generate with N beams), ...].
    Returns the filled token rows [nb, len(seq)]."""
    tokenizer = get_tokenizer(args)
    device = seq.device
    assert len(seq.shape) == 1
    tmpl = seq.tolist()
    out_seq_length = len(tmpl)
    n_img = tokenizer.img_tokenizer.num_tokens
    roi2 = tokenizer['[ROI2]']

    def slices_after(tok, cur):
        return _slices_after(tokenizer, tok, cur)

    context_length, offset, invalid_slices = _scan_context(tmpl, tokenizer)
    tokens, attention_mask, position_ids = get_batch(seq[:context_length], device, args)

    counter = context_length - 1
    index = 0
    if mems is None:
        mems = []
    score = [0]
    is_sparse = getattr(args, 'is_sparse', 0)
    if is_sparse == 2:
        img_indices_bool = tokens < n_img
        txt_indices_bool = ~img_indices_bool
    elif is_sparse == 0:
        txt_indices_bool = img_indices_bool = None
    else:
        raise ValueError('set is_sparse==2 for inference.')

    while counter < out_seq_length - 1:
        nxt = tmpl[counter + 1]
        invalid_slices = slices_after(nxt, invalid_slices)
        if index == 0:      # first call: the whole context
            position_ids = position_ids.clone()
            position_ids[position_ids > offset] -= offset
            logits, *mems = model(tokens, position_ids, attention_mask, txt_indices_bool, img_indices_bool, is_sparse,
                                  *mems)
            index = counter
        elif nxt >= 0:      # provided token
            if nxt == roi2:
                offset = counter + 1
            tokens, mems, score = shrink_beams(tokens, mems, 1, score)
            counter += 1
            tokens = torch.cat((tokens, seq[counter: counter + 1].expand(tokens.shape[0], 1)), dim=1)
            if is_sparse == 2:
                img_indices_bool = tokens < n_img
                txt_indices_bool = ~img_indices_bool
            continue
        else:
            assert tokens.shape[1] == counter + 1
            # A stretch of identical 'generate' slots: run it with the sampling tail inside the decode graph (no host
            # work per token).  Same operations as the loop body below; falls through when it does not apply.
            run = 1
            while counter + 1 + run < out_seq_length and tmpl[counter + 1 + run] == nxt:
                run += 1
            first_pos = counter - offset if counter > offset else counter
            device_pivots = is_sparse == 2 and _os.environ.get('COGVIEW_B200_SPARSE_PIVOTS', 'device') != 'host'
            # nucleus sampling of a single row keeps the host loop (and torch.multinomial's draws)
            if (run >= 2 and index == counter and tokens.shape[0] == -nxt
                    and (args.top_p == 0.0 or tokens.shape[0] > 1)
                    and (is_sparse == 0 or device_pivots)
                    and not (counter <= offset < counter + run) and hasattr(model, 'generate_run')):
                sparse = dict(n_img=n_img, tokens=tokens) if is_sparse == 2 else None
                nucleus = dict(top_p=args.top_p) if args.top_p > 0.0 else {}
                res = model.generate_run(tokens[:, counter:], first_pos, mems, run, args.temperature, args.top_k,
                                         invalid_slices, sparse=sparse, **nucleus)
                if res is not None:
                    new_tokens, logp, mems = res
                    if -nxt > 1:
                        score = (score if torch.is_tensor(score) else torch.tensor(score, device=device)) + logp
                    tokens = torch.cat((tokens, new_tokens), dim=1)
                    if is_sparse == 2:
                        img_indices_bool = tokens < n_img
                        txt_indices_bool = ~img_indices_bool
                    counter += run
                    index = counter
                    continue
            position_ids = torch.arange(index, counter + 1, dtype=torch.long, device=device).unsqueeze(0)
            position_ids[position_ids > offset] -= offset
            tokens, mems, score = shrink_beams(tokens, mems, -nxt, score)
            logits, *mems = model(tokens[:, index:], position_ids, 0, txt_indices_bool, img_indices_bool, is_sparse,
                                  *mems)
            index = counter
        nb = -nxt
        counter += 1
        index += 1

        log_probs = _next_token_probs(logits, invalid_slices, args)

        if nb > 1 and tokens.shape[0] == 1:     # 1 -> nb beams
            tokens = tokens.expand(nb, -1).contiguous()
            mems = [mem.expand(nb, -1, -1) for mem in mems]
            prev = torch.multinomial(log_probs, num_samples=nb, replacement=True)
            score = torch.log(torch.gather(log_probs, dim=1, index=prev)[0])
        else:
            assert tokens.shape[0] == nb
            prev = torch.multinomial(log_probs, num_samples=1)
            if nb > 1:      # beam scores are only consulted when beams shrink: keep them on the device
                score_plus = torch.log(torch.gather(log_probs, dim=1, index=prev)[:, 0])
                score = (score if torch.is_tensor(score) else torch.tensor(score, device=device)) + score_plus
        tokens = torch.cat((tokens, prev.view(tokens.shape[0], 1)), dim=1)
        if is_sparse == 2:
            img_indices_bool = tokens < n_img
            txt_indices_bool = ~img_indices_bool
    return tokens.view(tokens.shape[0], -1).contiguous()


def _batch_plan(model, tmpls, args, tokenizer):
    """Per template (context length, [ROI2] offset, beam count, generate slots), and whether filling_sequences can
    run all of them as one decode batch: every template is a context followed by one run of at least three generate
    slots of the same beam count, to its end; all share the slot count, the beam count and the invalid slices; dense
    attention on the K|V cache without nucleus sampling; at most ops.DECODE_MAX_BATCH rows; and the graph-replayed
    decode path is on."""
    from .. import ops
    plans, keys = [], set()
    ok = (getattr(args, 'is_sparse', 0) == 0 and args.top_p == 0.0 and hasattr(model, 'generate_run')
          and not torch.is_grad_enabled())
    for tmpl in tmpls:
        C, offset, inv = _scan_context(tmpl, tokenizer)
        gen = tmpl[C:]
        nb = -gen[0] if gen else 0
        plans.append((C, offset, nb, len(gen)))
        keys.add((nb, len(gen), tuple((sl.start, sl.stop) for sl in inv)))
        run = len(gen) - 1              # the first slot is drawn from the prompt's own forward
        ok = ok and C > 0 and nb > 0 and run >= 2 and all(x == -nb for x in gen) and not (C <= offset < C + run)
    tr = getattr(model, 'transformer', None)
    rows = sum(p[2] for p in plans)
    ok = (ok and len(keys) == 1 and tr is not None and getattr(tr, 'mems_mode', None) == 'kv'
          and rows <= ops.DECODE_MAX_BATCH and ops.decode_batch_supported(rows, tr.hidden_size)
          and max(p[0] for p in plans) + plans[0][3] - 1 <= tr.max_memory_length
          and _os.environ.get('COGVIEW_B200_FAST_DECODE', '1') != '0'
          and _os.environ.get('COGVIEW_B200_GRAPH_SAMPLING', '1') != '0')
    return plans, ok


def _stretches(tmpl, C, tokenizer):
    """The part of a template after its context C as (structure, given, slices): structure is the tuple of
    (given run length, generate run length, beam count) pairs in order (the first given run is empty: the context
    ends where the first generate slot starts) followed by the length of a trailing given run; given[s] the provided
    tokens before generate stretch s (given[-1]: the trailing ones); slices[s] the invalid vocabulary slices in force
    at generate stretch s, as filling_sequence tracks them."""
    _, _, inv = _scan_context(tmpl, tokenizer)
    structure, given, slices = [], [], []
    i, n, g0 = C, len(tmpl), C
    while i < n:
        g0 = i
        while i < n and tmpl[i] >= 0:
            inv = _slices_after(tokenizer, tmpl[i], inv)
            i += 1
        if i == n:
            break
        nb = tmpl[i]
        k0 = i
        while i < n and tmpl[i] == nb:
            i += 1
        structure.append((k0 - g0, i - k0, -nb))
        given.append(tmpl[g0:k0])
        slices.append(inv)
    given.append(tmpl[g0:] if i == n and g0 < n and tmpl[n - 1] >= 0 else [])
    structure.append(len(given[-1]))
    return tuple(structure), given, slices


def _stretch_plan(model, tmpls, args, tokenizer):
    """Per template (context length, [ROI2] offset, (structure, given, slices) of _stretches), and whether
    filling_sequences can run all of them as one decode batch with given stretches between the generate stretches
    (super-resolution windows: each 32-code line is given codes, then generated ones): every template has at least
    two generate stretches, all share one structure (the same given / generate run lengths in the same order, one
    beam each) and the invalid slices at every generate stretch; the given tokens and the context length are each
    template's own.  Plus the conditions of _batch_plan: dense attention on the K|V cache without nucleus sampling,
    at most ops.DECODE_MAX_BATCH rows, the longest context plus the rest of the template within max_memory_length,
    the graph-replayed decode path on."""
    from .. import ops
    plans, keys = [], set()
    ok = (getattr(args, 'is_sparse', 0) == 0 and args.top_p == 0.0 and hasattr(model, 'generate_run')
          and hasattr(model, 'chunk_run') and not torch.is_grad_enabled())
    for tmpl in tmpls:
        C, offset, _ = _scan_context(tmpl, tokenizer)
        st = _stretches(tmpl, C, tokenizer)
        plans.append((C, offset, st))
        structure, _, slices = st
        keys.add((structure, tuple(tuple((sl.start, sl.stop) for sl in inv) for inv in slices)))
        ok = ok and C > 0 and len(structure) >= 3 and all(nb == 1 for _, _, nb in structure[:-1])
    tr = getattr(model, 'transformer', None)
    rows = len(tmpls)
    ok = (ok and len(keys) == 1 and tr is not None and getattr(tr, 'mems_mode', None) == 'kv'
          and rows <= ops.DECODE_MAX_BATCH and ops.decode_batch_supported(rows, tr.hidden_size)
          and max(p[0] for p in plans) + len(tmpls[0]) - plans[0][0] - 1 <= tr.max_memory_length
          and _os.environ.get('COGVIEW_B200_FAST_DECODE', '1') != '0'
          and _os.environ.get('COGVIEW_B200_GRAPH_SAMPLING', '1') != '0')
    return plans, ok


def _row_positions(pos, offsets):
    """Absolute positions [b, n] -> model position ids: positions after a row's [ROI2] restart from it
    (position_ids[position_ids > offset] -= offset, per row)."""
    off = torch.as_tensor(offsets, dtype=torch.long, device=pos.device).view(-1, 1).expand_as(pos)
    return torch.where(pos > off, pos - off, pos)


def _fill_interleaved(model, seqs, tmpls, plans, args, tokenizer):
    """filling_sequences for templates that passed _stretch_plan: one row per template.  Each context is prefilled
    alone and its first generated token drawn as filling_sequence draws it; its cache goes straight into its row of
    the batch cache (kv_cache.assemble_rows, row_pad); then per generate stretch: the pending sampled token plus the given run go
    through GPT2Model.chunk_run (in pieces of at most ops.ATTN_CHUNK_MAX tokens), the stretch's first slot is drawn
    from its logits, and the rest of the stretch runs through generate_run on the ragged decode graph."""
    from .. import ops
    from ..mpu import kv_cache
    device = seqs[0].device
    roi2 = tokenizer['[ROI2]']
    structure, _, slices = plans[0][2]
    ctx = [p[0] for p in plans]
    offsets = [p[1] for p in plans]
    out = [seq.clone().view(1, -1) for seq in seqs]
    last = []

    def prefill(r):
        tokens, attention_mask, position_ids = get_batch(seqs[r][:ctx[r]], device, args)
        position_ids = position_ids.clone()
        position_ids[position_ids > offsets[r]] -= offsets[r]
        logits, *mems = model(tokens, position_ids, attention_mask, None, None, 0)
        last.append(torch.multinomial(_next_token_probs(logits, slices[0], args), num_samples=1))
        return mems
    mems, row_pad = kv_cache.assemble_rows(model.transformer, ctx, [1] * len(seqs), len(tmpls[0]) - ctx[0] - 1,
                                           prefill)
    last = torch.cat(last, dim=0)
    ctx_t = torch.tensor(ctx, dtype=torch.long, device=device).view(-1, 1)
    rel = 0                                                  # template slot (after the context) of `last`
    for s, (g, k, _) in enumerate(structure[:-1]):
        if s > 0:
            given = torch.tensor([p[2][1][s] for p in plans], dtype=torch.long, device=device)
            for r, p in enumerate(plans):                    # a given [ROI2] restarts that row's positions
                for e, tok in enumerate(p[2][1][s]):
                    if tok == roi2:
                        offsets[r] = ctx[r] + rel + 1 + e
            chunk = torch.cat((last.to(device), given), dim=1)
            pos = _row_positions(ctx_t + torch.arange(rel, rel + g + 1, device=device).view(1, -1), offsets)
            for c0 in range(0, g + 1, ops.ATTN_CHUNK_MAX):
                res = model.chunk_run(chunk[:, c0:c0 + ops.ATTN_CHUNK_MAX], pos[:, c0:c0 + ops.ATTN_CHUNK_MAX],
                                      mems, row_pad)
                if res is None:
                    raise RuntimeError('filling_sequences: the chunk of %d rows was refused' % chunk.shape[0])
                logits, mems = res
            rel += g + 1
            last = torch.multinomial(_next_token_probs(logits.unsqueeze(1), slices[s], args), num_samples=1)
        for r, o in enumerate(out):
            o[0, ctx[r] + rel] = last[r, 0]
        if k > 1:
            first_pos = _row_positions(ctx_t + rel, offsets).view(-1)
            res = model.generate_run(last, first_pos, mems, k - 1, args.temperature, args.top_k, slices[s],
                                     row_pad=row_pad)
            if res is None:
                raise RuntimeError('filling_sequences: the decode batch of %d rows was refused' % last.shape[0])
            new_tokens, _, mems = res
            for r, o in enumerate(out):
                o[0, ctx[r] + rel + 1:ctx[r] + rel + k] = new_tokens[r].to(device)
            last = new_tokens[:, -1:]
        rel += k - 1
    return out


def filling_sequences(model, seqs, args):
    """filling_sequence for several templates (1-D LongTensors, e.g. one per caption) at once: returns one token tensor
    [nb, len(seq_c)] per template.  Each context is run through the model on its own (batch 1) and its nb first tokens
    are drawn as filling_sequence draws them; then the generate slots of all rows run as ONE decode batch (DecodeRunner
    in ragged mode: every row continues at its own context length and position).  Templates that interleave given
    and generated stretches with one beam each (super-resolution windows, see _stretch_plan) share a batch too: the
    given stretches go through GPT2Model.chunk_run, every row at its own cache length.  Templates that cannot share a
    batch (see _batch_plan and _stretch_plan) are filled one by one with filling_sequence, as is a single template.
    The abs-max LayerNorm scales of the decode step and of the chunk are taken over the whole batch, so a template's
    rows match a run of that template alone within bf16 tolerance, not bit for bit."""
    if len(seqs) == 1:
        return [filling_sequence(model, seqs[0], args)]
    tokenizer = get_tokenizer(args)
    tmpls = [seq.tolist() for seq in seqs]
    plans, ok = _batch_plan(model, tmpls, args, tokenizer)
    if not ok:
        splans, sok = _stretch_plan(model, tmpls, args, tokenizer)
        if sok:
            return _fill_interleaved(model, seqs, tmpls, splans, args, tokenizer)
        return [filling_sequence(model, seq, args) for seq in seqs]
    from ..mpu import kv_cache
    device = seqs[0].device
    prefixes, first_pos = [], []
    _, _, invalid_slices = _scan_context(tmpls[0], tokenizer)     # shared by all templates (_batch_plan)

    def prefill(c):
        C, offset, nb, _ = plans[c]
        tokens, attention_mask, position_ids = get_batch(seqs[c][:C], device, args)
        position_ids = position_ids.clone()
        position_ids[position_ids > offset] -= offset
        logits, *mems = model(tokens, position_ids, attention_mask, None, None, 0)
        probs = _next_token_probs(logits, invalid_slices, args)
        prev = torch.multinomial(probs, num_samples=nb, replacement=True) if nb > 1 else torch.multinomial(probs, 1)
        prefixes.append(torch.cat((tokens.expand(nb, -1), prev.view(nb, 1)), dim=1))
        first_pos.extend([C - offset if C > offset else C] * nb)
        return mems
    run = plans[0][3] - 1
    # each prompt's K|V goes into its rows of the batch cache before the next prompt reuses the batch-1 cache
    mems, row_pad = kv_cache.assemble_rows(model.transformer, [p[0] for p in plans], [p[2] for p in plans], run,
                                           prefill)
    last = torch.cat([p[:, -1:] for p in prefixes], dim=0)
    res = model.generate_run(last, first_pos, mems, run, args.temperature, args.top_k, invalid_slices,
                             row_pad=row_pad)
    if res is None:
        raise RuntimeError('filling_sequences: the decode batch of %d rows was refused' % last.shape[0])
    new_tokens = res[0]
    out, r0 = [], 0
    for p in prefixes:
        nb = p.shape[0]
        out.append(torch.cat((p, new_tokens[r0:r0 + nb].to(p.device)), dim=1))
        r0 += nb
    return out


def _completion_plan(model, tmpls, args, tokenizer):
    """The decode window of every template for filling_completions, and whether it can run them as one decode batch.
    Template r's first and last generate slots are f_r and l_r; S = max_r (l_r - f_r + 1) is the number of decode
    steps; row r's window starts at c_r = max(2, l_r + 1 - S) <= f_r.  Its tokens [0, c_r - 1) are prefilled; decode
    step j feeds token c_r - 1 + j and yields slot c_r + j, so the S steps cover slots c_r .. c_r + S - 1, which hold
    every generate slot of the row; the given tokens among them are forced, those after them only copied.
    Returns (plans, S, ok): plans[r] = (c_r, beam count, [ROI2] offset of the prefill, invalid slices).  The
    conditions: every template has generate slots, all of one beam count, with the same invalid slices at each of
    them in every template; no [ROI2] among the fed tokens; the window inside the template and the cache; dense
    attention on the K|V cache; at most ops.DECODE_MAX_BATCH rows (and a hidden size the decode kernels take at that
    batch); not a single row with nucleus sampling (filling_sequence's host loop keeps its torch.multinomial draws);
    the graph-replayed decode path on."""
    from .. import ops
    roi2 = tokenizer['[ROI2]']
    spans, slice_keys = [], set()
    ok = (getattr(args, 'is_sparse', 0) == 0 and hasattr(model, 'generate_run') and not torch.is_grad_enabled())
    for tmpl in tmpls:
        gen = [i for i, x in enumerate(tmpl) if x < 0]
        if not gen or len({tmpl[i] for i in gen}) != 1:
            return [], 0, False
        _, _, slices = _stretches(tmpl, gen[0], tokenizer)
        slice_keys.update(tuple((sl.start, sl.stop) for sl in inv) for inv in slices)
        spans.append((gen[0], gen[-1], -tmpl[gen[0]], slices[0]))
    S = max(l - f + 1 for f, l, _, _ in spans)
    plans = []
    for tmpl, (f, l, nb, inv) in zip(tmpls, spans):
        c = max(2, l + 1 - S)
        ok = ok and c <= f and c + S <= len(tmpl) and roi2 not in tmpl[c - 1:c + S - 1]
        offset = max([i for i, x in enumerate(tmpl[:c - 1]) if x == roi2], default=100000)
        plans.append((c, nb, offset, inv))
    tr = getattr(model, 'transformer', None)
    rows = sum(p[1] for p in plans)
    ok = (ok and len(slice_keys) == 1 and tr is not None and getattr(tr, 'mems_mode', None) == 'kv'
          and rows <= ops.DECODE_MAX_BATCH and ops.decode_batch_supported(rows, tr.hidden_size)
          and max(p[0] for p in plans) - 1 + S <= tr.max_memory_length
          and not (rows == 1 and args.top_p > 0.0)
          and _os.environ.get('COGVIEW_B200_FAST_DECODE', '1') != '0'
          and _os.environ.get('COGVIEW_B200_GRAPH_SAMPLING', '1') != '0')
    return plans, S, ok


def filling_completions(model, seqs, args):
    """filling_sequences for templates whose given and generate slots differ from template to template (images
    completed under a different mask each, see generate.complete_images): returns one token tensor [nb, len(seq_c)]
    per template.  Templates that filling_sequences batches (one layout for all: a context then one generate run, or
    the interleaved stretches of _stretch_plan) go there.  Otherwise every row runs the window of _completion_plan:
    its tokens before the window are prefilled alone at batch 1 into its rows of the batch cache
    (kv_cache.assemble_rows, row_pad), then all rows run S = max_r (l_r - f_r + 1) steps as ONE ragged graph-replayed
    decode (GPT2Model.generate_run with `forced`): at a generate slot a row keeps its draw, at a given slot the given
    token replaces it, and either is the next step's input.  A template's nb rows share its prefill and are drawn
    independently of each other (filling_sequence instead keeps the best-scoring beam at each given token after
    generated ones); no beam scores are kept.  With top_p > 0 the nucleus filter runs in the sampling kernel.
    Templates _completion_plan refuses are filled one by one with filling_sequence.  The abs-max LayerNorm scales of
    the decode step are taken over the whole batch, so a row matches a run of its template alone within bf16
    tolerance, not bit for bit."""
    tokenizer = get_tokenizer(args)
    tmpls = [seq.tolist() for seq in seqs]
    if len(seqs) > 1 and (_batch_plan(model, tmpls, args, tokenizer)[1]
                          or _stretch_plan(model, tmpls, args, tokenizer)[1]):
        return filling_sequences(model, seqs, args)
    plans, S, ok = _completion_plan(model, tmpls, args, tokenizer)
    if not ok:
        return [filling_sequence(model, seq, args) for seq in seqs]
    from ..mpu import kv_cache
    device = seqs[0].device

    def prefill(r):
        c, _, offset, _ = plans[r]
        tokens, attention_mask, position_ids = get_batch(seqs[r][:c - 1], device, args)
        position_ids = position_ids.clone()
        position_ids[position_ids > offset] -= offset
        _, *mems = model(tokens, position_ids, attention_mask, None, None, 0, logits_last_only=True)
        return mems
    mems, row_pad = kv_cache.assemble_rows(model.transformer, [p[0] - 1 for p in plans], [p[1] for p in plans], S,
                                           prefill)
    rows = [(tmpl, c, offset) for tmpl, (c, nb, offset, _) in zip(tmpls, plans) for _ in range(nb)]
    last = torch.tensor([[tmpl[c - 1]] for tmpl, c, _ in rows], dtype=torch.long, device=device)
    first_pos = [c - 1 - offset if c - 1 > offset else c - 1 for _, c, offset in rows]
    forced = torch.tensor([[max(x, -1) for x in tmpl[c:c + S]] for tmpl, c, _ in rows], dtype=torch.long,
                          device=device)
    res = model.generate_run(last, first_pos, mems, S, args.temperature, args.top_k, plans[0][3], row_pad=row_pad,
                             top_p=args.top_p, forced=forced)
    if res is None:
        raise RuntimeError('filling_completions: the decode batch of %d rows was refused' % len(rows))
    new_tokens = res[0].to(device)
    out, r0 = [], 0
    for seq, (c, nb, _, _) in zip(seqs, plans):
        filled = seq.view(1, -1).repeat(nb, 1)
        filled[:, c:c + S] = new_tokens[r0:r0 + nb]
        out.append(filled)
        r0 += nb
    return out


def _shared_plan(model, tmpls, args, tokenizer):
    """_batch_plan, and whether filling_shared_prompts can run the templates: _batch_plan's conditions (for one
    template too), every context of the same length, and a model with shared_run."""
    plans, ok = _batch_plan(model, tmpls, args, tokenizer)
    return plans, ok and len({p[0] for p in plans}) == 1 and hasattr(model, 'shared_run')


def filling_shared_prompts(model, seqs, args):
    """filling_sequences for templates whose prompts are long next to what is generated (image2text: a 1028-token
    image prompt, 20 text slots): returns one token tensor [nb, len(seq_c)] per template.  All contexts go through ONE
    GPT2Model.forward at batch len(seqs) (logits of the last position only), whose K|V cache is the prefix every beam of
    a template reads; the nb first tokens of each template are drawn from its prompt's logits as filling_sequence draws
    them; the remaining slots run as one graph-replayed decode batch in which each prompt's K|V is read once for all of
    its beams (GPT2Model.shared_run, cv_attn_decode_shared).  Needs the conditions of _batch_plan and contexts of one
    length (_shared_plan); otherwise the templates go to filling_sequences.  The abs-max LayerNorm scales of the
    prompt forward and of the decode step are taken over the whole batch, so a template's rows match a run of that
    template alone within bf16 tolerance, not bit for bit."""
    tokenizer = get_tokenizer(args)
    tmpls = [seq.tolist() for seq in seqs]
    plans, ok = _shared_plan(model, tmpls, args, tokenizer)
    if not ok:
        return filling_sequences(model, seqs, args)
    device = seqs[0].device
    C, offset, nb, n_gen = plans[0]
    _, _, invalid_slices = _scan_context(tmpls[0], tokenizer)     # shared by all templates (_batch_plan)
    tokens = torch.stack([seq[:C] for seq in seqs]).to(device)
    attention_mask, _, position_ids = get_masks_and_position_ids(tokens)
    position_ids = position_ids.clone()
    position_ids[position_ids > offset] -= offset
    logits, *mems = model(tokens, position_ids, attention_mask, None, None, 0, logits_last_only=True)
    probs = _next_token_probs(logits, invalid_slices, args)
    prev = torch.multinomial(probs, num_samples=nb, replacement=True)          # [templates, nb]
    res = model.shared_run(prev.reshape(-1, 1), C - offset if C > offset else C, mems, n_gen - 1, args.temperature,
                           args.top_k, invalid_slices)
    if res is None:
        raise RuntimeError('filling_shared_prompts: the decode batch of %d rows was refused' % prev.numel())
    new_tokens = res[0].to(device)
    return [torch.cat((tokens[i].expand(nb, -1), prev[i].view(nb, 1), new_tokens[i * nb:(i + 1) * nb]), dim=1)
            for i in range(len(seqs))]


def inverse_prompt_score(model, seq, args):
    """generation/sampling.py:214-230 — caption log-likelihood given the image (post-selection)."""
    tokenizer = get_tokenizer(args)
    device = seq.device
    assert len(seq.shape) == 2
    botext = 2 + 1024 + 1
    assert tokenizer['[ROI1]'] == seq[0][botext]
    tokens, attention_mask, position_ids = get_batch(seq, device, args)
    logits, *mems = model(tokens, position_ids, attention_mask, None, None, getattr(args, 'is_sparse', 0))
    logits[..., :tokenizer.img_tokenizer.num_tokens] = -float('Inf')
    log_probs = torch.log(F.softmax(logits, dim=-1))
    pred = log_probs[:, botext:-1, :]
    target = tokens[:, botext + 1:].unsqueeze(-1)
    return torch.gather(pred, dim=2, index=target).squeeze(-1).sum(dim=-1)


def inverse_prompt_scores(model, seqs, args):
    """inverse_prompt_score for many post-selection rows at once, on GPT2Model.token_logprobs: the caption
    log-likelihood given the image of every row, fp32 [N] in input order.  seqs: a 2-D LongTensor or a list of 1-D
    rows ([BASE] [BOI1] 1024 codes [EOI1] [ROI1] caption); rows may belong to different captions, so their lengths may
    differ.  Rows go through the model in groups of at most args.max_inference_batch_size, each group padded at the
    end with [PAD] (causal attention keeps the padding out of every scored position).  Each caption token is scored
    over the vocabulary window [img_tokenizer.num_tokens, V), the window the reference's -inf mask leaves.  No logits
    and no K|V cache are kept.  The abs-max LayerNorm scale is one scalar per forward tensor, so a row of a mixed or
    padded group matches a run of that row alone within bf16 tolerance, not bit for bit; where the reference's fp32
    log(softmax) underflows to -inf, this returns the finite log-probability.  Dense attention (is_sparse=0) only."""
    if getattr(args, 'is_sparse', 0) != 0:
        raise NotImplementedError('inverse_prompt_scores supports dense attention (is_sparse=0) only')
    tokenizer = get_tokenizer(args)
    rows = list(seqs.unbind(0)) if torch.is_tensor(seqs) else list(seqs)
    botext = 2 + 1024 + 1
    assert all(r.dim() == 1 and r.shape[0] > botext + 1 for r in rows), 'post-selection rows hold a caption'
    n = len(rows)
    mbz = max(1, args.max_inference_batch_size)
    n_img = tokenizer.img_tokenizer.num_tokens
    pad, roi1 = tokenizer['[PAD]'], tokenizer['[ROI1]']
    out = []
    with torch.no_grad():
        for g0 in range(0, n, mbz):
            group = rows[g0:g0 + mbz]
            device = group[0].device
            lens = [r.shape[0] for r in group]
            L = max(lens)
            tokens = torch.full((len(group), L), pad, dtype=torch.long, device=device)
            for i, r in enumerate(group):
                tokens[i, :lens[i]] = r.to(device)
            assert bool((tokens[:, botext] == roi1).all()), 'post-selection rows have [ROI1] at index %d' % botext
            attention_mask, _, position_ids = get_masks_and_position_ids(tokens)
            # row i scores positions botext .. lens[i] - 2, each predicting the token after it
            ncap = torch.tensor([n_ - 1 - botext for n_ in lens], device=device)
            col = torch.arange(max(lens) - 1 - botext, device=device).view(1, -1)
            valid = col < ncap.view(-1, 1)
            flat = (torch.arange(len(group), device=device).view(-1, 1) * L + botext + col)[valid]
            lp = model.token_logprobs(tokens, position_ids, attention_mask, flat, tokens.view(-1)[flat + 1],
                                      vocab_begin=n_img)
            per_pos = torch.zeros(valid.shape, dtype=torch.float32, device=lp.device)
            per_pos[valid.to(lp.device)] = lp
            out.append(per_pos.sum(dim=1))        # in position order per row: no atomics, the same sum every call
    return torch.cat(out, dim=0)
