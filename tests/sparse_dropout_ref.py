"""Test helpers for the attention-probability dropout of sparse training attention (no GPU needed to import):

* `sparse_attention_keep`: the oracle's sparse_attention (oracle/cogview_oracle.py, mpu/sparse_transformer.py:675-725) with
  dropout applied where the reference applies it (:719-721): probs * keep / (1 - p) after the joint softmax.  keep is a
  [b, heads, s, n_piv + w*times] 0/1 tensor in the reference's probability layout (pivot columns, then window columns);
  with keep = None it is the oracle unchanged.
* `keep_layout` / `decode_keep`: the keep-bit buffer of cv_attn_sparse_fwd with dropout (layout in
  include/cogview_b200.h) decoded into per-(query, virtual key) decisions, and converted to the reference layout by
  `to_reference_layout`.
"""
import math

import torch
import torch.nn.functional as F

from oracle import cogview_oracle as O

T = 128


def sparse_attention_keep(q, k, v, pivot_idx, pivot_attention_mask, query_window=128, key_window_times=6, keep=None,
                          dropout_p=0.0):
    b, n_head, s, hn = q.shape
    n_piv = pivot_idx.shape[1]
    w, times = query_window, key_window_times
    gidx = pivot_idx.view(b, 1, n_piv, 1).expand(b, n_head, n_piv, hn)
    pk, pv = torch.gather(k, 2, gidx), torch.gather(v, 2, gidx)
    pm = pivot_attention_mask.unsqueeze(1)
    sp = torch.matmul(q, pk.transpose(-1, -2)) * (pm / math.sqrt(hn)) - 10000.0 * (1.0 - pm)
    sp = sp + math.log(s // n_piv)
    if s % w != 0:
        raise ValueError('The seq_len must be exactly divided by window_size.')
    wk, wv = O._overlapping_windows(k, w, times), O._overlapping_windows(v, w, times)
    wq = q.view(b, n_head, s // w, w, hn)
    sw = torch.matmul(wq, wk.transpose(-1, -2))
    wm = torch.ones((w, w * times), dtype=sw.dtype).tril_(diagonal=w * (times - 1))
    sw = sw * (wm / math.sqrt(hn)) - 10000.0 * (1.0 - wm)
    sw = sw.clone()
    for t in range(1, times):
        sw[:, :, t - 1, :, :w * times - w * t] -= 10000.0
    sw = sw.view(b, n_head, s, w * times)
    probs = torch.softmax(torch.cat((sp, sw), dim=-1), dim=-1)
    if keep is not None:
        probs = probs * keep / (1.0 - dropout_p)
    ctx_p = torch.matmul(probs[..., :n_piv], pv)
    ctx_w = torch.einsum('bcgwk,bcgkh->bcgwh', probs[..., n_piv:].view(b, n_head, s // w, w, w * times), wv)
    return ctx_p + ctx_w.reshape(b, n_head, s, hn)


def band_start(i, w, times):
    return max(0, i // w - times + 1) * w


def keep_layout(b, heads, s, n_piv, w, times):
    """The tile walk of include/cogview_b200.h (cv_attn_sparse_fwd with dropout) restated in Python."""
    nqb = nkb = (s + T - 1) // T
    npb = (n_piv + T - 1) // T
    last = [min(qb * T + T, s) - 1 for qb in range(nqb)]
    jb0 = [band_start(qb * T, w, times) // T for qb in range(nqb)]
    nband = [last[qb] // T - jb0[qb] + 1 for qb in range(nqb)]
    sees_piv = [band_start(last[qb], w, times) > 0 for qb in range(nqb)]
    i_end = [min(nqb - 1, (((kb * T + T - 1) // w + times) * w - 1) // T) for kb in range(nkb)]
    piv0 = (times * w) // T
    L = dict(nqb=nqb, nkb=nkb, npb=npb, jb0=jb0, nband=nband, sees_piv=sees_piv, i_end=i_end, piv0=piv0,
             tb=max(nband), tq=max(i_end[kb] - kb + 1 for kb in range(nkb)), np=nqb - piv0 if times * w < s else 0)
    L["words"] = (b * heads * nqb * T * (L["tb"] + npb) * 4, b * heads * nkb * T * L["tq"] * 4,
                  b * heads * npb * T * L["np"] * 4)
    return L


def _bits(words, shape):
    """int32 words [..., 4] -> 0/1 uint8 [..., 128] (bit t of word g = entry 32g + t)."""
    w = words.cpu().to(torch.int64).view(*shape, 4) & 0xFFFFFFFF
    return ((w.unsqueeze(-1) >> torch.arange(32)) & 1).to(torch.uint8).reshape(*shape, 128)


def decode_keep(mask, b, heads, s, n_piv, w, times):
    """Returns (fwd, bwd): int8 [b, heads, s, nkb*128 + npb*128] decisions over the virtual keys (band keys, then pivot
    slots) as the forward / the backward passes read them; -1 where that kernel reads nothing."""
    L = keep_layout(b, heads, s, n_piv, w, times)
    nqb, nkb, npb = L["nqb"], L["nkb"], L["npb"]
    fw, bw, pw = L["words"]
    assert mask.numel() == fw + bw + pw, (mask.numel(), L["words"])
    flat = mask.view(-1)
    fbits = _bits(flat[:fw], (b, heads, nqb * T, L["tb"] + npb))
    nv = (nkb + npb) * T
    fwd = torch.full((b, heads, nqb * T, nv), -1, dtype=torch.int8)
    bwd = torch.full((b, heads, nqb * T, nv), -1, dtype=torch.int8)
    for qb in range(nqb):
        rows = slice(qb * T, qb * T + T)
        for j in range(L["nband"][qb]):
            kb = L["jb0"][qb] + j
            fwd[:, :, rows, kb * T:kb * T + T] = fbits[:, :, rows, j].to(torch.int8)
        if L["sees_piv"][qb]:
            for pb in range(npb):
                c = (nkb + pb) * T
                fwd[:, :, rows, c:c + T] = fbits[:, :, rows, L["nband"][qb] + pb].to(torch.int8)
    if bw:
        bbits = _bits(flat[fw:fw + bw], (b, heads, nkb * T, L["tq"]))     # [.., key, slot, query in block]
        for kb in range(nkb):
            for u in range(L["i_end"][kb] - kb + 1):
                qb = kb + u
                bwd[:, :, qb * T:qb * T + T, kb * T:kb * T + T] = \
                    bbits[:, :, kb * T:kb * T + T, u].transpose(-1, -2).to(torch.int8)
    if pw:
        pbits = _bits(flat[fw + bw:], (b, heads, npb * T, L["np"]))
        for pb in range(npb):
            c = (nkb + pb) * T
            for u in range(L["np"]):
                qb = L["piv0"] + u
                bwd[:, :, qb * T:qb * T + T, c:c + T] = pbits[:, :, pb * T:pb * T + T, u].transpose(-1, -2).to(torch.int8)
    return fwd[:, :, :s], bwd[:, :, :s]


def visible(s, n_piv, w, times, pivot_idx):
    """bool [b, s, nkb*128 + npb*128]: the (query, virtual key) pairs the sparse attention gives a nonzero weight."""
    b = pivot_idx.shape[0]
    nkb, npb = (s + T - 1) // T, (n_piv + T - 1) // T
    i = torch.arange(s).view(s, 1)
    bs = torch.tensor([band_start(x, w, times) for x in range(s)]).view(s, 1)
    j = torch.arange(nkb * T).view(1, -1)
    band = ((j >= bs) & (j <= i)).unsqueeze(0).expand(b, s, nkb * T)
    pos = torch.full((b, npb * T), 1 << 40, dtype=torch.int64)
    pos[:, :n_piv] = pivot_idx
    piv = pos.unsqueeze(1) < bs.view(1, s, 1)
    return torch.cat((band, piv), dim=-1)


def to_reference_layout(fwd, s, n_piv, w, times):
    """[b, heads, s, virtual keys] decisions -> [b, heads, s, n_piv + w*times] float keep (window column c of query i is
    key (i // w - times + 1) * w + c; entries the attention masks out are set to 1)."""
    b, heads = fwd.shape[:2]
    nkb = (s + T - 1) // T
    i = torch.arange(s).view(s, 1)
    key = (i // w - times + 1) * w + torch.arange(w * times).view(1, -1)
    win = fwd[:, :, :, :nkb * T].gather(-1, key.clamp_min(0).view(1, 1, s, -1).expand(b, heads, s, w * times).long())
    win = torch.where((key >= 0) & (key <= i), win, torch.ones_like(win))
    piv = fwd[:, :, :, nkb * T:nkb * T + n_piv]
    keep = torch.cat((piv, win), dim=-1).float()
    return keep.clamp_min(0)     # unwritten pivot entries are only those of queries that see no pivot (masked)
