"""generate.super_resolution (generate_samples.py:223-244) with stand-ins for the model's `fill` and the VQ-VAE's
`decode`: the template is split as the reference splits it (last 1024 tokens = the 32 x 32 source codes, the rest =
the text prefix), the 4096 magnified codes reach the decoder as one 64 x 64 grid, and debug=True puts the source
image, decoded and interpolated to 512 x 512, first."""
import torch
import torch.nn.functional as F


def _tok():
    from cogview_b200.generation import sampling
    return sampling.TokenLayout(img_tokens=8192, txt_tokens=101)


def _query(tok, seed=0):
    from cogview_b200 import generate
    g = torch.Generator().manual_seed(seed)
    text = (8192 + torch.randint(0, 101, (6,), generator=g)).tolist()
    src = torch.randint(0, 8192, (1024,), generator=g).tolist()
    seq = generate.build_query(generate.QUERY_TEMPLATES['super-resolution'], [text, src], tokenizer=tok)
    return torch.tensor(seq, dtype=torch.long), text, src


def _fake_decode(calls):
    def decode(codes):
        calls.append(codes.clone())
        b, h, w = codes.shape
        # a per-pixel pattern that depends on the codes, so that the interpolation and the order are visible
        base = codes.float().repeat_interleave(8, 1).repeat_interleave(8, 2).unsqueeze(1)
        return torch.cat((base, base + 0.25, base + 0.5), dim=1)
    return decode


def test_super_resolution_splits_the_template_and_decodes_one_64x64_grid(monkeypatch):
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    tok = _tok()
    monkeypatch.setattr(sampling, "_TOKENIZER", tok)
    seq, text, src = _query(tok)
    assert seq[:len(text) + 3].tolist() == [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']]
    magnified = torch.randint(0, 8192, (1, 4096), generator=torch.Generator().manual_seed(1))
    seen = {}

    def fake_magnify(model, tokenizer, tokens_list, text_token_list, args, fill=None):
        seen.update(tokenizer=tokenizer, codes=tokens_list.clone(), text=text_token_list.clone(), fill=fill)
        return magnified.clone()
    monkeypatch.setattr(generate, "magnify", fake_magnify)
    calls = []

    def fill(model, seq, args, invalid_slices=None):
        raise AssertionError("not reached: magnify is replaced")
    codes, imgs = generate.super_resolution(torch.nn.Identity(), None, None, seq, fill=fill, decode=_fake_decode(calls))
    assert seen["tokenizer"] is tok and seen["fill"] is fill
    assert seen["codes"].tolist() == src                                   # seq[-1024:]
    assert seen["text"].tolist() == seq[:-1024].tolist()                   # seq[:-1024]
    assert seen["text"].tolist() == [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']]
    assert torch.equal(codes, magnified)
    assert len(calls) == 1 and calls[0].shape == (1, 64, 64) and torch.equal(calls[0].view(1, 4096), magnified)
    assert imgs.shape == (1, 3, 512, 512)
    assert torch.equal(imgs, _fake_decode([])(magnified.view(1, 64, 64)))


def test_super_resolution_debug_puts_the_interpolated_source_first(monkeypatch):
    from cogview_b200 import generate
    from cogview_b200.generation import magnify as mg
    from cogview_b200.generation import sampling
    tok = _tok()
    monkeypatch.setattr(sampling, "_TOKENIZER", tok)
    seq, text, src = _query(tok, seed=2)
    windows = []

    def fake_fill(model, s, args, invalid_slices=None):      # "generates" code (row * 64 + col) % 8192 at (row, col)
        i, j, line = mg.WINDOWS[len(windows)]
        windows.append((i, j))
        ctx = len(seq) - 1024 + 256 + 5
        assert s.shape[0] == ctx + line * 32
        assert torch.equal(s[:len(seq) - 1024], seq[:-1024])
        rows = torch.arange(16 * i, 16 * i + line).view(-1, 1)
        cols = torch.arange(16 * j, 16 * j + 32).view(1, -1)
        part = torch.where(s[ctx:].view(line, 32) < 0, (rows * 64 + cols) % 8192, s[ctx:].view(line, 32))
        return torch.cat((s[:ctx], part.reshape(-1))).unsqueeze(0)
    calls = []
    codes, imgs = generate.super_resolution(torch.nn.Identity(), None, None, seq, fill=fake_fill,
                                            decode=_fake_decode(calls), debug=True)
    assert len(windows) == 9
    assert torch.equal(codes.view(64, 64), torch.arange(4096).view(64, 64) % 8192)
    assert [c.shape for c in calls] == [(1, 32, 32), (1, 64, 64)]
    assert calls[0].view(-1).tolist() == src and torch.equal(calls[1].view(1, -1), codes)
    assert imgs.shape == (2, 3, 512, 512)
    src_img = _fake_decode([])(torch.tensor(src).view(1, 32, 32))
    assert torch.equal(imgs[:1], F.interpolate(src_img, size=(512, 512)))
    assert torch.equal(imgs[1:], _fake_decode([])(codes.view(1, 64, 64)))
