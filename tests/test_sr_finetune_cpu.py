"""Host side of finetuning the super-resolution model: the finetune position ids (positions restart at each row's
first [ROI2], then clamp to the position table) against the reference's per-row loop written out here, the two-image
rows of make_super_resolution_batch with a stand-in encoder, and the rows' round trip through a BinaryDataset file
into make_batch."""
import random
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cogview_b200 import data as D
from cogview_b200.generation import sampling
from cogview_b200.generation.sampling import get_masks_and_position_ids

TOK = sampling.TokenLayout()        # 8192 image codes + 50000 text pieces + 27 command tokens
ROI2 = TOK['[ROI2]']
MPE, MPE_FT = 1089, 2121
FT = types.SimpleNamespace(finetune=True, max_position_embeddings=MPE, max_position_embeddings_finetune=MPE_FT)
PW = [0, 128, 256] * 3
PH = [0, 0, 0, 128, 128, 128, 256, 256, 256]


@pytest.fixture(autouse=True)
def _tokenizer(monkeypatch):
    monkeypatch.setattr(sampling, "_TOKENIZER", TOK)


def reference_positions(data, max_position_embeddings):
    """pretrain_gpt2.py:228-247, the reference's finetune branch as it is written."""
    batch_size, seq_length = data.size()
    tmp = torch.nonzero(data == ROI2, as_tuple=False)
    start_token_poses = [100000] * batch_size
    for x, y in tmp:
        start_token_poses[x] = min(start_token_poses[x], y)
    assert 100000 not in start_token_poses, 'Some samples do not have [ROI2]!'
    position_ids = torch.zeros(batch_size, seq_length, dtype=torch.long)
    for i in range(batch_size):
        sep = start_token_poses[i]
        torch.arange(start=0, end=sep, out=position_ids[i, :sep], dtype=torch.long)
        torch.arange(start=0, end=seq_length - sep, out=position_ids[i, sep:], dtype=torch.long)
    position_ids[position_ids >= max_position_embeddings] = max_position_embeddings - 1
    return position_ids


def sr_row(n_text, pose, seed):
    """A row with the layout make_super_resolution_batch writes: [ROI1] text [BASE] [BOI1] 1024 codes [EOI1] [ROI2]
    [POSi] [BASE] [BOI2] 1024 codes [EOI2]."""
    g = torch.Generator().manual_seed(seed)
    text = (8192 + torch.randint(0, 50000, (n_text,), generator=g)).tolist()
    c0, c1 = torch.randint(0, 8192, (2, 1024), generator=g).tolist()
    return ([TOK['[ROI1]']] + text + [TOK['[BASE]'], TOK['[BOI1]']] + c0 +
            [TOK['[EOI1]'], ROI2, TOK['[POS%d]' % pose], TOK['[BASE]'], TOK['[BOI2]']] + c1 + [TOK['[EOI2]']])


# ----------------------------------------------------------------------------------------------------
# finetune position ids
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens", [(60, 61), (62, 64), (3, 64), (0, 10)])
def test_positions_equal_reference_loop_on_rows(lens):
    """Rows of T + 2057 tokens padded to 2121 (tokens are the first 2120): with T = 60 and 61 the first segment just
    fits the 1089-entry table, from T = 62 on its tail is clamped to 1088."""
    rows = [sr_row(t, 4, seed=t) for t in lens]
    text = torch.full((len(rows), MPE_FT), TOK['[PAD]'], dtype=torch.long)
    for i, r in enumerate(rows):
        text[i, :len(r)] = torch.tensor(r)
    tokens = text[:, :-1]
    _, _, pos = get_masks_and_position_ids(tokens, args=FT)
    ref = reference_positions(tokens, MPE)
    assert pos.dtype == torch.long and torch.equal(pos, ref)
    for i, t in enumerate(lens):
        sep = t + 1028
        assert tokens[i, sep] == ROI2 and pos[i, sep] == 0 and pos[i, sep + 1] == 1
        assert int(pos[i, :sep].max()) == min(sep - 1, MPE - 1)
        assert int(pos.max()) <= MPE - 1


def test_positions_roi2_anywhere_first_wins_and_clamp():
    """Short rows with a small table: [ROI2] at the start, in the middle, at the end, twice (the first one restarts
    the positions, the second is an ordinary token), with the clamp cutting into both segments."""
    args = types.SimpleNamespace(finetune=True, max_position_embeddings=6, max_position_embeddings_finetune=16)
    g = torch.Generator().manual_seed(0)
    data = torch.randint(0, 8192, (6, 16), generator=g)
    for r, cols in enumerate([[0], [5], [15], [3, 9], [9, 3], [7, 8]]):
        data[r, cols] = ROI2
    _, _, pos = get_masks_and_position_ids(data, args=args)
    assert torch.equal(pos, reference_positions(data, 6))
    assert pos[3, 3] == 0 and pos[3, 9] == 5 and pos[4, 3] == 0
    assert pos[1].tolist() == [0, 1, 2, 3, 4, 0, 1, 2, 3, 4, 5, 5, 5, 5, 5, 5]


def test_positions_missing_roi2_raises():
    data = torch.randint(0, 8192, (3, 32), generator=torch.Generator().manual_seed(1))
    data[0, 4] = ROI2
    data[2, 30] = ROI2
    with pytest.raises(AssertionError, match=r"Some samples do not have \[ROI2\]!"):
        get_masks_and_position_ids(data, args=FT)


@pytest.mark.parametrize("args", [None, types.SimpleNamespace(finetune=False, max_position_embeddings=MPE,
                                                             max_position_embeddings_finetune=MPE_FT),
                                  types.SimpleNamespace(finetune=True, max_position_embeddings=MPE,
                                                        max_position_embeddings_finetune=MPE)])
def test_positions_without_the_finetune_branch_are_arange(args):
    data = torch.randint(0, 8192, (2, 40), generator=torch.Generator().manual_seed(2))
    data[:, 7] = ROI2
    lm = torch.rand(2, 40)
    mask, loss_mask, pos = get_masks_and_position_ids(data, loss_mask=lm, args=args)
    m0, l0, p0 = get_masks_and_position_ids(data, loss_mask=lm)
    assert torch.equal(pos, torch.arange(40).unsqueeze(0).expand_as(data)) and torch.equal(pos, p0)
    assert torch.equal(mask, m0) and mask.shape == (1, 1, 40, 40) and loss_mask is lm


# ----------------------------------------------------------------------------------------------------
# make_super_resolution_batch with a stand-in encoder
# ----------------------------------------------------------------------------------------------------
class Encode:
    """Records the images it is given; image k of the call encodes to (k * 1024 + arange(1024)) % 8192."""

    def __init__(self):
        self.calls = []

    def __call__(self, x):
        self.calls.append(x.clone())
        return (torch.arange(x.shape[0]).view(-1, 1) * 1024 + torch.arange(1024).view(1, -1)) % 8192


def _images(n, seed=0):
    return torch.randn((n, 3, 512, 512), generator=torch.Generator().manual_seed(seed))


def test_builder_layout_poses_and_crops():
    n, k = 3, 4
    texts = [[8192 + 5 * i + j for j in range(t)] for i, t in enumerate([7, 1, 64])]
    imgs = _images(n)
    enc = Encode()
    random.seed(11)
    want_poses = random.choices(range(9), weights=[1] * 9, k=k)
    random.seed(11)
    rows = D.make_super_resolution_batch(None, texts, imgs, sampling_num=k, encode=enc)
    assert len(enc.calls) == 1, "one batched encoder call"
    x = enc.calls[0]
    assert x.shape == (n + n * k, 3, 256, 256)
    assert torch.equal(x[:n], F.interpolate(imgs, size=(256, 256), mode='bilinear'))
    codes = enc(x)
    assert len(rows) == n * k
    for i in range(n):
        for j in range(k):
            row = rows[i * k + j]
            T = len(texts[i])
            assert row.dtype == torch.int64 and row.dim() == 1 and len(row) == T + 2057
            r = row.tolist()
            assert r[:T + 3] == [TOK['[ROI1]']] + texts[i] + [TOK['[BASE]'], TOK['[BOI1]']]
            assert r[T + 3:T + 1027] == codes[i].tolist()
            p = want_poses[j]
            assert r[T + 1027:T + 1032] == [TOK['[EOI1]'], ROI2, TOK['[POS%d]' % p], TOK['[BASE]'], TOK['[BOI2]']]
            assert r[T + 1032:T + 2056] == codes[n + i * k + j].tolist()
            assert r[-1] == TOK['[EOI2]']
            assert torch.equal(x[n + i * k + j], imgs[i, :, PH[p]:PH[p] + 256, PW[p]:PW[p] + 256])


def test_builder_poses_shared_and_reproducible():
    imgs = _images(2, seed=1)
    texts = [[8200], [8300, 8301]]

    def poses(rows):
        return [[int(r[len(t) + 1029]) - TOK['[POS0]'] for r in rows[i * 6:(i + 1) * 6]] for i, t in enumerate(texts)]
    random.seed(3)
    a = poses(D.make_super_resolution_batch(None, texts, imgs, sampling_num=6, encode=Encode()))
    random.seed(3)
    b = poses(D.make_super_resolution_batch(None, texts, imgs, sampling_num=6, encode=Encode()))
    assert a == b and a[0] == a[1]
    assert all(0 <= p < 9 for p in a[0])
    draws = set()
    for s in range(20):
        random.seed(100 + s)
        draws.add(tuple(poses(D.make_super_resolution_batch(None, texts, imgs, sampling_num=6, encode=Encode()))[0]))
    assert len(draws) > 1


def test_builder_refuses_other_sizes():
    with pytest.raises(NotImplementedError):
        D.make_super_resolution_batch(None, [[8200]], torch.zeros(1, 3, 256, 256), img_size=256, encode=Encode())
    with pytest.raises(ValueError):
        D.make_super_resolution_batch(None, [[8200], [8201]], torch.zeros(1, 3, 512, 512), encode=Encode())


# ----------------------------------------------------------------------------------------------------
# storage: write_tokenized_rows -> BinaryDataset -> filled_tokenized_process_fn -> make_batch
# ----------------------------------------------------------------------------------------------------
def test_storage_round_trip(tmp_path):
    rows = [torch.tensor(sr_row(t, p, seed=t)) for t, p in [(64, 0), (5, 8), (60, 3)]]
    path = str(tmp_path / "sr.bin")
    assert D.write_tokenized_rows(path, rows, MPE_FT) == 3
    raw = np.fromfile(path, dtype=np.int32).reshape(3, MPE_FT)
    for r, w in zip(rows, raw):
        assert np.array_equal(w[:len(r)], r.numpy()) and (w[len(r):] == -1).all()
    ds = D.BinaryDataset(path, D.filled_tokenized_process_fn(MPE_FT), length_per_sample=MPE_FT)
    assert len(ds) == 3
    items = [ds[i] for i in range(3)]
    for r, it in zip(rows, items):
        n = len(r)
        assert it['text'].dtype == np.int64 and len(it['text']) == MPE_FT
        assert np.array_equal(it['text'][:n], r.numpy()) and (it['text'][n:] == TOK['[PAD]']).all()
        assert it['loss_mask'].tolist() == [1] * n + [0] * (MPE_FT - n)
    batch = {k: np.stack([it[k] for it in items]) for k in ('text', 'loss_mask')}
    tokens, labels, loss_mask, mask, pos = D.make_batch(batch, args=FT)
    text = torch.from_numpy(batch['text'])
    assert tokens.shape == labels.shape == loss_mask.shape == pos.shape == (3, MPE_FT - 1)
    assert torch.equal(tokens, text[:, :-1]) and torch.equal(labels, text[:, 1:])
    for i, r in enumerate(rows):
        assert loss_mask[i].tolist() == [1.0] * (len(r) - 1) + [0.0] * (MPE_FT - len(r))
    assert torch.equal(pos, reference_positions(tokens, MPE))
    assert mask.shape == (1, 1, MPE_FT - 1, MPE_FT - 1)
    _, _, _, _, pos0 = D.make_batch(batch)
    assert torch.equal(pos0, torch.arange(MPE_FT - 1).unsqueeze(0).expand(3, -1))


def test_write_refuses_long_rows(tmp_path):
    with pytest.raises(ValueError):
        D.write_tokenized_rows(str(tmp_path / "x.bin"), [list(range(10))], 8)
