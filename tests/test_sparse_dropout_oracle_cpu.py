"""Host-side checks of the sparse-attention dropout test helpers (tests/sparse_dropout_ref.py): the dropout-aware oracle
reduces to the pinned oracle when nothing is dropped, applies keep / (1 - p) to the joint probabilities, and the Python
restatement of the keep-bit buffer layout sizes it exactly as the library does."""
import pytest
import torch

from oracle import cogview_oracle as O
import sparse_dropout_ref as R


def _inputs(b, nh, s, w, times, n_piv, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn((b, nh, s, 64), generator=g) for _ in range(3))
    pivot_idx = torch.stack([torch.randperm(s, generator=g)[:n_piv].sort().values for _ in range(b)])
    bs = torch.tensor([R.band_start(i, w, times) for i in range(s)])
    pam = (pivot_idx.unsqueeze(1) < bs.view(1, s, 1)).float()      # the closed form of the gathered rmask
    return q, k, v, pivot_idx, pam


def test_keep_none_is_the_oracle_and_keep_scales_the_probabilities():
    b, nh, s, w, times, n_piv = 2, 2, 256, 32, 3, 40
    q, k, v, pivot_idx, pam = _inputs(b, nh, s, w, times, n_piv, 0)
    ref = O.sparse_attention(q, k, v, pivot_idx, pam, w, times)
    assert torch.equal(R.sparse_attention_keep(q, k, v, pivot_idx, pam, w, times), ref)
    ones = torch.ones((b, nh, s, n_piv + w * times))
    assert torch.equal(R.sparse_attention_keep(q, k, v, pivot_idx, pam, w, times, keep=ones, dropout_p=0.0), ref)
    # keep = 1 everywhere with p = 0.5 doubles every probability (exactly: a power of two)
    assert torch.equal(R.sparse_attention_keep(q, k, v, pivot_idx, pam, w, times, keep=ones, dropout_p=0.5), 2 * ref)
    # dropping every pivot column leaves the band part of the same joint softmax
    nopiv = ones.clone()
    nopiv[..., :n_piv] = 0
    out = R.sparse_attention_keep(q, k, v, pivot_idx, pam, w, times, keep=nopiv, dropout_p=0.0)
    late = s - w                                                       # queries that see pivots
    assert not torch.allclose(out[:, :, late:], ref[:, :, late:])
    assert torch.allclose(out[:, :, :w * times], ref[:, :, :w * times])   # no query here sees a pivot


@pytest.mark.parametrize("b,heads,s,n_piv,w,times", [(2, 3, 512, 96, 64, 3), (1, 2, 1024, 200, 128, 6),
                                                     (1, 40, 4096, 768, 128, 6), (2, 1, 256, 40, 128, 2),
                                                     (1, 1, 320, 20, 64, 5), (3, 2, 448, 64, 64, 2)])
def test_keep_buffer_size_matches_the_library(b, heads, s, n_piv, w, times):
    from cogview_b200 import _lib
    L = R.keep_layout(b, heads, s, n_piv, w, times)
    assert _lib.lib().cv_attn_sparse_drop_mask_words(b, heads, s, n_piv, w, times) == sum(L["words"])
    if (s, n_piv, w, times) == (4096, 768, 128, 6):
        per_seq_head = sum(L["words"]) * 4 / (b * heads)
        print("keep bits at s=4096, w=128, times=6, 768 pivots: %.2f MB per (sequence, head)" % (per_seq_head / 2 ** 20))
        assert per_seq_head < 2 * 2 ** 20
