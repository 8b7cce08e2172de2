"""K|V-cache form of the reference's `mems` (mpu/sparse_transformer.py:526-529, :615-626).

The reference caches per-layer HIDDEN STATES and re-normalises / re-projects the whole memory every step
(:320, :136-141).  In 'kv' mode the list returned by GPT2Model.forward has the same length (num_layers + 1)
and the same batch / time axes, but entry i (< num_layers) is a view [b, t, 2h] of layer i's key|value cache
and the last entry is an empty placeholder; `filling_sequence` only ever expands / slices the batch axis and
passes the list back, which both forms support.  The cache buffers are pre-allocated to max_memory_length
and appended in place (positions >= t only, so an older view stays valid).
"""
import torch


class _Caches:
    def __init__(self, owner, b, device):
        self.h = owner.hidden_size
        self.L = len(owner.layers)
        self.maxlen = owner.max_memory_length
        self.b = b
        self.t = 0
        self.buf = torch.empty((self.L, b, self.maxlen, 2 * self.h), dtype=torch.bfloat16, device=device)
        self.dummy = torch.empty((b, self.maxlen, 0), dtype=torch.bfloat16, device=device)
        self.sq = 0

    def matches(self, mems, b):
        """True if `mems` are exactly this cache's current views (so we can append in place)."""
        if len(mems) != self.L + 1 or b != self.b:
            return False
        m0 = mems[0]
        return (m0.data_ptr() == self.buf[0].data_ptr() and m0.shape[0] == b and m0.shape[2] == 2 * self.h
                and m0.stride(0) == self.buf.stride(1) and m0.stride(1) == self.buf.stride(2))

    def load_from(self, mems):
        t = mems[0].size(1)
        for i in range(self.L):
            self.buf[i, :, :t].copy_(mems[i])
        self.t = t

    def begin(self, sq):
        if self.t + sq > self.maxlen:
            raise NotImplementedError('KV-cache overflow: memory %d + %d new tokens > max_memory_length %d '
                                      '(sliding memories need mems_mode="hidden")' % (self.t, sq, self.maxlen))
        self.sq = sq

    def appender(self, i):
        t, sq, h = self.t, self.sq, self.h
        layer_buf = self.buf[i]

        def kv(k_new, v_new):
            layer_buf[:, t:t + sq, :h].copy_(k_new)
            layer_buf[:, t:t + sq, h:].copy_(v_new)
            cur = layer_buf[:, :t + sq]
            return cur[..., :h], cur[..., h:]
        return kv

    def views(self):
        self.t += self.sq
        out = [self.buf[i, :, :self.t] for i in range(self.L)]
        out.append(self.dummy[:, :self.t])
        return out


# Caches of several batch sizes are kept so that a run that alternates between them (one prompt, then its beams)
# does not re-allocate and re-capture; but at the 4B shape a 32-sequence and a 64-sequence cache together are 51 GB.
# When the pooled caches would exceed this many bytes, those of the other batch sizes are dropped first.  It holds a
# 64-row cache of the 4B shape at max_memory_length 1345 (super-resolution windows: 39.4 GiB) together with the batch-1
# cache its prompts are prefilled in (0.6 GiB), so the two are not dropped and re-made in turn for every window.
POOL_BYTE_BUDGET = 41 << 30


def cache_bytes(owner, b):
    return len(owner.layers) * b * owner.max_memory_length * 2 * owner.hidden_size * 2


def _make_room(owner, pool, b, need=None, keep=()):
    """Called before a cache for batch size b (or pool key b) is allocated: drop pooled caches of other sizes, largest
    first, until the pool with the new cache of `need` bytes (default: cache_bytes) fits POOL_BYTE_BUDGET (the new
    cache itself is always allowed).  The keys in `keep` are counted but not dropped."""
    need = cache_bytes(owner, b) if need is None else need
    total = need + sum(pool[k].buf.numel() * 2 for k in pool if k != b)
    others = sorted((k for k in pool if k != b and k not in keep), key=lambda k: pool[k].buf.numel(), reverse=True)
    for k in others:
        if total <= POOL_BYTE_BUDGET:
            break
        total -= pool[k].buf.numel() * 2
        if getattr(owner, '_kv', None) is pool[k]:
            owner._kv = None
        # the cache and its DecodeRunner refer to each other: break the cycle so that the cache's memory is returned
        # now, not at the next garbage collection (a new cache of another size is about to be allocated)
        pool[k].runner = None
        del pool[k]


def _pooled(owner, b):
    """(pool, the pooled cache of batch size b or None); room for a new one is made when there is none."""
    dev = owner.position_embeddings.weight.device
    pool = owner.__dict__.setdefault('_kv_pool', {})
    c = pool.get(b)
    if c is not None and (c.maxlen != owner.max_memory_length or c.buf.device != dev):
        c = None
        del pool[b]
    if c is None:
        _make_room(owner, pool, b)
    return pool, c, dev


def prepare(owner, mems, b, sq):
    """Find (or build) the cache that `mems` refers to and get it ready for sq more tokens.  One cache (and its
    captured decode graph) is kept per batch size and reused across sequences, within POOL_BYTE_BUDGET."""
    pool, c, dev = _pooled(owner, b)
    if not mems:
        if c is None:
            c = _Caches(owner, b, dev)
        c.t = 0
    elif c is not None and c.matches(mems, b):
        c.t = mems[0].size(1)
    else:
        # beams were expanded / selected (generation/sampling.py:168-172, :188-198): copy into this batch size's cache
        if c is None:
            c = _Caches(owner, b, dev)
        c.load_from(mems)
    pool[b] = c
    owner._kv = c
    c.begin(sq)
    return c


def assemble(owner, caption_mems, rows, run):
    """The cache of one decode batch whose rows come from prompts of different lengths.  caption_mems[c] is prompt
    c's `mems` at batch 1 (len_c tokens, as GPT2Model.forward returned them); its K|V fills slots [0, len_c) of the
    next rows[c] rows of the pooled cache of batch size sum(rows).  Returns (mems of that batch, t = max(len_c) tokens
    long, row_pad int32 [b] on the device = t - len_c of every row): the decode continues row i at its own length
    t - row_pad[i] (DecodeRunner's ragged mode).  Slots past a row's own length are left as they were."""
    lens = [m[0].size(1) for m in caption_mems]
    t = max(lens)
    if t + run > owner.max_memory_length:
        raise NotImplementedError('KV-cache overflow: longest prompt %d + %d new tokens > max_memory_length %d'
                                  % (t, run, owner.max_memory_length))
    b = sum(rows)
    pool, c, dev = _pooled(owner, b)
    if c is None:
        c = _Caches(owner, b, dev)
    r0 = 0
    for mems, n, ln in zip(caption_mems, rows, lens):
        assert len(mems) == c.L + 1 and mems[0].size(0) == 1
        for i in range(c.L):
            c.buf[i, r0:r0 + n, :ln].copy_(mems[i].expand(n, -1, -1))
        r0 += n
    c.t = t
    pool[b] = c
    owner._kv = c
    row_pad = torch.tensor([t - ln for ln, n in zip(lens, rows) for _ in range(n)], dtype=torch.int32, device=dev)
    return [c.buf[i, :, :t] for i in range(c.L)] + [c.dummy[:, :t]], row_pad


def assemble_rows(owner, lens, rows, run, prefill):
    """assemble without holding every prompt's cache at once (super-resolution windows have contexts of ~800 tokens:
    64 copies of such a batch-1 cache take as much memory as the batch cache itself).  prefill(c) runs prompt c at
    batch 1 and returns its `mems` (lens[c] tokens); they are copied into the next rows[c] rows of the pooled cache of
    batch size sum(rows) before the next prompt runs.  Same cache contents and return value as assemble."""
    t = max(lens)
    if t + run > owner.max_memory_length:
        raise NotImplementedError('KV-cache overflow: longest prompt %d + %d new tokens > max_memory_length %d'
                                  % (t, run, owner.max_memory_length))
    b = sum(rows)
    c, r0 = None, 0
    for ci, (n, ln) in enumerate(zip(rows, lens)):
        mems = prefill(ci)
        assert mems[0].size(0) == 1 and mems[0].size(1) == ln
        if c is None:           # after the first prompt, whose batch-1 cache is then already pooled
            pool, c, dev = _pooled(owner, b)
            if c is None:
                c = _Caches(owner, b, dev)
            pool[b] = c
        for i in range(c.L):
            c.buf[i, r0:r0 + n, :ln].copy_(mems[i].expand(n, -1, -1))
        r0 += n
    c.t = t
    pool[b] = c
    owner._kv = c
    row_pad = torch.tensor([t - ln for ln, n in zip(lens, rows) for _ in range(n)], dtype=torch.int32,
                           device=c.buf.device)
    return [c.buf[i, :, :t] for i in range(c.L)] + [c.dummy[:, :t]], row_pad


class _SharedCaches:
    """The generated tokens of a decode batch whose rows share prompts (DecodeRunner's shared mode): b rows in `groups`
    groups of G = b / groups consecutive rows.  Group g's prompt K|V is row g of the pooled cache of batch size groups
    (`prefix`, P tokens, filled by one forward over the prompts and only read by the decode); row r's generated
    tokens go to buf[:, r, :maxlen]."""

    def __init__(self, owner, b, groups, run, device):
        self.h = owner.hidden_size
        self.L = len(owner.layers)
        self.b, self.groups, self.maxlen = b, groups, run
        self.buf = torch.empty((self.L, b, run, 2 * self.h), dtype=torch.bfloat16, device=device)
        self.prefix, self.P = None, 0
        self.runner = None


def shared(owner, prefix, P, b, run):
    """The suffix cache of b rows continuing the prefix.b prompts of the pooled cache `prefix` (P tokens each), with room
    for `run` tokens per row.  It is pooled under ('shared', b, groups, run) with its DecodeRunner, so the next batch of
    the same shape reuses both, and its bytes count against POOL_BYTE_BUDGET; the prefix cache is never dropped to
    make room for it.  The caller sets .prefix back to None after the run, so that the suffix cache does not keep a
    prefix cache alive that the pool has since dropped."""
    assert b % prefix.b == 0 and 0 < P and P <= prefix.maxlen and run >= 1
    pool = owner.__dict__.setdefault('_kv_pool', {})
    assert pool.get(prefix.b) is prefix
    key = ('shared', b, prefix.b, run)
    c = pool.get(key)
    if c is not None and c.buf.device != prefix.buf.device:
        c = None
        del pool[key]
    if c is None:
        _make_room(owner, pool, key, need=len(owner.layers) * b * run * 2 * owner.hidden_size * 2, keep=(prefix.b,))
        c = pool[key] = _SharedCaches(owner, b, prefix.b, run, prefix.buf.device)
    c.prefix, c.P = prefix, P
    return c
