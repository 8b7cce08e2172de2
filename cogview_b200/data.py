"""Data formats feeding the training path (SURVEY §8(f) rank 4): the compact binary token files and the
text+code template of the reference.

  BinaryDataset              data_utils/datasets.py:63-81      [N, 64 + 1024] int32 rows, memory-mapped
  compact_binary_process_fn  data_utils/datasets.py:119-128    row -> {'text', 'loss_mask'}
  TextCodeTemplate           data_utils/templates.py:52-65     [ROI1] text [BASE] [BOI1] code [EOI1]
  pad_to_len                 data_utils/datasets.py:91-101
  make_batch                 pretrain_gpt2.py:256-289          tokens / labels / loss mask / attention mask / positions
  make_super_resolution_batch  preprocess/pretokenized_data.py:89-140   two-image super-resolution finetune rows
  write_tokenized_rows / filled_tokenized_process_fn                   those variable-length rows in a BinaryDataset

Host-side numpy / torch, apart from the VQ-VAE encoding of make_super_resolution_batch; LMDB datasets and
sentencepiece stay out of scope (synthetic or pre-tokenised text)."""
import random

import numpy as np
import torch
import torch.nn.functional as F

from . import vqvae
from .generation.sampling import get_masks_and_position_ids, get_tokenizer


def TextCodeTemplate(text, code, tokenizer=None):
    """data_utils/templates.py:52-65 for already-tokenised text (numpy array or list of ids)."""
    tok = tokenizer or get_tokenizer()
    if isinstance(text, str):
        raise NotImplementedError('raw strings need the sentencepiece tokenizer, which is outside this package')
    code = tok.wrap_code(code)
    if isinstance(text, list) and isinstance(code, list):
        return [tok['[ROI1]']] + text + code
    return np.concatenate((np.array([tok['[ROI1]']]), np.asarray(text), np.asarray(code)), axis=0)


def pad_to_len(ret, max_len, tokenizer=None):
    """data_utils/datasets.py:91-101: right-pad with [PAD] (or truncate) to max_len; returns (row, valid length)."""
    tok = tokenizer or get_tokenizer()
    if len(ret) < max_len:
        return np.concatenate((ret, np.array([tok['[PAD]']] * (max_len - len(ret)))), axis=0), len(ret)
    return ret[:max_len], max_len


def compact_binary_process_fn(max_len, tokenizer=None):
    """data_utils/datasets.py:119-128: 64 text slots (-1 = unused) + 1024 image codes per row."""
    def process_fn(row):
        text, code = row[:64].astype(np.int64), row[64:].astype(np.int64)
        text = text[text > -1]
        ret, sep = pad_to_len(TextCodeTemplate(text, code, tokenizer), max_len, tokenizer)
        return {'text': ret, 'loss_mask': np.array([1] * sep + [0] * (len(ret) - sep))}
    return process_fn


def tokenized_process_fn(max_len, tokenizer=None):
    """data_utils/datasets.py:103-109: rows that were tokenised when saved."""
    def process_fn(row):
        ret, sep = pad_to_len(row.flatten(), max_len, tokenizer)
        return {'text': ret, 'loss_mask': np.array([1] * sep + [0] * (len(ret) - sep))}
    return process_fn


def filled_tokenized_process_fn(max_len, tokenizer=None):
    """tokenized_process_fn for rows shorter than the file's row length (write_tokenized_rows): the -1 fill is
    stripped, then the row is padded with [PAD] to max_len and its loss mask covers the row's own tokens only."""
    def process_fn(row):
        row = row.flatten()
        ret, sep = pad_to_len(row[row > -1].astype(np.int64), max_len, tokenizer)
        return {'text': ret, 'loss_mask': np.array([1] * sep + [0] * (len(ret) - sep))}
    return process_fn


def write_tokenized_rows(path, rows, length_per_sample):
    """Write token rows of any length up to length_per_sample as the int32 [N, length_per_sample] file BinaryDataset
    reads, each row filled up with -1 (read back with filled_tokenized_process_fn).  Returns the row count."""
    out = np.full((len(rows), length_per_sample), -1, dtype=np.int32)
    for i, r in enumerate(rows):
        r = np.asarray(r.cpu() if torch.is_tensor(r) else r).reshape(-1)
        if len(r) > length_per_sample:
            raise ValueError('row %d has %d tokens, more than length_per_sample = %d' % (i, len(r), length_per_sample))
        if len(r) and (r.min() < 0 or r.max() > np.iinfo(np.int32).max):
            raise ValueError('row %d holds a token id outside [0, 2^31)' % i)
        out[i, :len(r)] = r
    out.tofile(path)
    return len(rows)


def make_super_resolution_batch(vq_model, texts, imgs, img_size=512, sampling_num=4, encode=None):
    """preprocess/pretokenized_data.py:89-140: the super-resolution finetune rows of N images.  texts: N lists of
    text ids, already in the unified vocabulary (what the reference's tokenizer(text) returns; sentencepiece stays
    with the caller).  imgs: [N, 3, 512, 512], normalised as vqvae.img2code takes them (the reference's read_img).
    `sampling_num` grid positions are drawn once per call with Python's random.choices and shared by every image;
    each image gives one row per drawn position, image-major:

        [ROI1] text [BASE] [BOI1] <overview, 1024 codes> [EOI1] [ROI2] [POSi] [BASE] [BOI2] <patch, 1024 codes> [EOI2]

    (len(text) + 2057 tokens), where the overview is the image bilinearly downsampled to 256 x 256 and the patch the
    256 x 256 crop at grid position i (rows and columns start at 0, 128 or 256).  All overviews and patches of the
    call go through one `encode` (default vqvae.img2code on vq_model).  Returns N * sampling_num int64 CPU rows."""
    if img_size != 512:
        raise NotImplementedError('super-resolution rows are built from 512 x 512 images only')
    tok = get_tokenizer()
    if imgs.dim() != 4 or tuple(imgs.shape[1:]) != (3, img_size, img_size):
        raise ValueError('imgs must be [N, 3, %d, %d], got %s' % (img_size, img_size, tuple(imgs.shape)))
    if len(texts) != imgs.shape[0]:
        raise ValueError('one text per image: %d texts, %d images' % (len(texts), imgs.shape[0]))
    encode = encode or (lambda x: vqvae.img2code(vq_model, x))
    t0, t1 = img_size // 4, img_size // 2
    pw = [0, t0, t1] * 3
    ph = [0, 0, 0, t0, t0, t0, t1, t1, t1]
    poses = random.choices(range(9), weights=[1] * 9, k=sampling_num)
    n = imgs.shape[0]
    patches = [imgs[i, :, ph[p]:ph[p] + t1, pw[p]:pw[p] + t1] for i in range(n) for p in poses]
    overviews = F.interpolate(imgs, size=(t1, t1), mode='bilinear')
    codes = encode(torch.cat((overviews, torch.stack(patches)), dim=0)).cpu().long()
    size_tk = tok['[BASE]']
    rows = []
    for i in range(n):
        head = torch.tensor([tok['[ROI1]']] + list(texts[i]) + [size_tk, tok['[BOI1]']], dtype=torch.long)
        for j, p in enumerate(poses):
            mid = torch.tensor([tok['[EOI1]'], tok['[ROI2]'], tok['[POS%d]' % p], size_tk, tok['[BOI2]']],
                               dtype=torch.long)
            rows.append(torch.cat((head, codes[i], mid, codes[n + i * sampling_num + j],
                                   torch.tensor([tok['[EOI2]']], dtype=torch.long))))
    return rows


class BinaryDataset(torch.utils.data.Dataset):
    """data_utils/datasets.py:63-81."""

    def __init__(self, path, process_fn, length_per_sample=64 + 1024, dtype='int32', preload=False, **kwargs):
        assert length_per_sample is not None
        self.length_per_sample = length_per_sample
        self.dtype = np.dtype(dtype)
        self.process_fn = process_fn
        if preload:
            self.bin = np.fromfile(path, dtype=self.dtype).reshape(-1, length_per_sample)
        else:
            with open(path, 'rb') as fid:
                flen = fid.seek(0, 2) // self.dtype.itemsize
            self.bin = np.memmap(path, dtype=self.dtype, mode='r',
                                 shape=(flen // length_per_sample, length_per_sample))

    def __len__(self):
        return self.bin.shape[0]

    def __getitem__(self, index):
        return self.process_fn(self.bin[index])


def make_batch(data, device=None, args=None):
    """pretrain_gpt2.py:256-289 without the model-parallel broadcast (MP = 1): `data` holds 'text' and 'loss_mask'
    [b, s + 1].  Returns tokens, labels, loss_mask, attention_mask, position_ids; `args` goes to
    get_masks_and_position_ids (its finetune branch restarts the positions at [ROI2])."""
    tokens_ = torch.as_tensor(np.asarray(data['text'])).long()
    loss_mask = torch.as_tensor(np.asarray(data['loss_mask'])).float()
    if device is not None:
        tokens_, loss_mask = tokens_.to(device), loss_mask.to(device)
    labels = tokens_[:, 1:].contiguous()
    loss_mask = loss_mask[:, 1:].contiguous()
    tokens = tokens_[:, :-1].contiguous()
    attention_mask, loss_mask, position_ids = get_masks_and_position_ids(tokens, loss_mask=loss_mask, args=args)
    return tokens, labels, loss_mask, attention_mask, position_ids
