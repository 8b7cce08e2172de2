"""Generation driver around `filling_sequence` — the token-level parts of generate_samples.py:68-200 and of
UnifiedTokenizer.parse_query / DecodeIds (data_utils/unified_tokenizer.py:91-196): query templates per task, query
assembly from already-tokenised text and image codes, beam batching, and decoding of the generated image codes
through the VQ-VAE.  Text <-> string conversion (sentencepiece) and image file I/O stay with the caller."""
from collections import namedtuple

import torch

from . import vqvae
from .generation.magnify import magnify, magnify_batch
from .generation.sampling import (add_interlacing_beam_marks, filling_completions, filling_sequence,
                                  filling_sequences, filling_shared_prompts, get_tokenizer, inverse_prompt_score,
                                  inverse_prompt_scores)

# generate_samples.py:203-214
QUERY_TEMPLATES = {
    'text2image': '[ROI1] {} [BASE] [BOI1] [MASK]*1024',
    'image2text': '[BASE] [BOI1] [Image]{} [EOI1] [ROI1] [MASK]*20',
    'low-level super-resolution': '[ROI1] {} [BASE] [BOI1] [Image]{} [EOI1] [ROI2] [POS0] [BASE] [BOI2] [MASK]*1024',
    'super-resolution': '[ROI1] {} [BASE] [BOI1] [Image]{}',
    'post-selection': '[BASE] [BOI1] [Image]{} [EOI1] [ROI1] {}',
}


def build_query(template, fields, tokenizer=None):
    """parse_query (data_utils/unified_tokenizer.py:154-196) for pre-tokenised fields.  `template` is one of
    QUERY_TEMPLATES' strings; each '{}' takes the next entry of `fields`: a list / 1-D tensor of text ids (already
    offset into the unified vocabulary) for a plain '{}', or of image codes for '[Image]{}' / '[ImageN]{}' (codes
    beyond N become -1 = to be generated).  '[MASK]' / '[MASK]*N' become -1 slots.  Returns a list of ints."""
    tok = tokenizer or get_tokenizer()
    fields = list(fields)
    ret = []
    for part in template.split(' '):
        if part == '[MASK]':
            ret.append(-1)
        elif part.startswith('[MASK]*'):
            c = int(part[7:])
            assert c > 0
            ret.extend([-1] * c)
        elif part.startswith('[Image'):
            num_codes, rest = part[6:].split(']')
            assert rest == '{}', 'image parts take their codes from `fields`'
            codes = [int(x) for x in fields.pop(0)]
            n = len(codes) if num_codes == '' else int(num_codes)
            ret.extend(codes[:n] + [-1] * (len(codes) - n))
        elif part == '{}':
            ret.extend(int(x) for x in fields.pop(0))
        elif part in tok.command_tokens:
            ret.append(tok[part])
        else:
            raise ValueError('raw text %r needs the sentencepiece tokenizer; pass token ids through `fields`' % part)
    assert not fields, 'more fields than placeholders'
    return ret


def split_tokens(ids, tokenizer=None):
    """DecodeIds (data_utils/unified_tokenizer.py:91-123) without the string / pixel decoders: returns (parts, images)
    where parts interleaves command-token names with lists of text ids (un-offset, as sentencepiece would get them)
    and images is the list of image-code lists, each closed by an [EOI*] token or the end of the row."""
    tok = tokenizer or get_tokenizer()
    names = {v: k for k, v in tok.command_tokens.items()}
    first_cmd = min(names)
    n_img = tok.img_tokenizer.num_tokens
    parts, images, img_buf, txt_buf = [], [], [], []
    for x in ids:
        x = int(x)
        if x >= first_cmd:
            name = names[x]
            if name.startswith('[EOI') and img_buf:
                images.append(img_buf)
                img_buf = []
            if txt_buf:
                parts.append(txt_buf)
                txt_buf = []
            parts.append(name)
        elif x < n_img:
            img_buf.append(x)
        else:
            txt_buf.append(x - n_img)
    if img_buf:
        images.append(img_buf)
    if txt_buf:
        parts.append(txt_buf)
    return parts, images


def generate_images_once(model, vq_model, args, seq, num=8, fill=filling_sequence, decode=None):
    """generate_samples.py:147-200 for the image-producing tasks: `num` samples of the template `seq` (1-D LongTensor
    with -1 slots) in groups of args.max_inference_batch_size beams; returns (token rows [num, len(seq)], images
    [num, 3, H, W]) where each image is the LAST image of its row (the generation target), decoded by the VQ-VAE."""
    decode = decode or (lambda codes: vqvae.code2img(vq_model, codes))
    mbz = args.max_inference_batch_size
    assert num < mbz or num % mbz == 0
    seq = seq.clone()
    add_interlacing_beam_marks(seq, nb=min(num, mbz))
    rows = []
    model.eval()
    with torch.no_grad():
        for _ in range(max(num // mbz, 1)):
            rows.append(fill(model, seq.clone(), args))
        rows = torch.cat(rows, dim=0)
        return rows, _decode_rows(rows, decode)


def _decode_rows(rows, decode):
    """The last image of every token row, decoded: [rows, 3, H, W]."""
    imgs = []
    for row in rows:
        _, images = split_tokens(row.tolist())
        codes = torch.tensor(images[-1], dtype=torch.long, device=rows.device).unsqueeze(0)
        img = decode(codes)
        if img.shape[-1] == 128:                       # low-level super-resolution sources are 128 x 128
            img = torch.nn.functional.interpolate(img, size=(256, 256))
        imgs.append(img)
    return torch.cat(imgs, dim=0)


def generate_images_batch(model, vq_model, args, seqs, num=8, fill=filling_sequences, decode=None):
    """generate_images_once for a list of templates (e.g. one per caption of a caption file): returns one
    (token rows [num, len(seq)], images [num, 3, H, W]) pair per template.  With num <= args.max_inference_batch_size
    whole templates are packed into decode batches of at most that many rows (`fill` takes a list of templates and
    returns a list of token tensors, see filling_sequences); above it every template runs through generate_images_once
    on its own."""
    decode = decode or (lambda codes: vqvae.code2img(vq_model, codes))
    mbz = args.max_inference_batch_size
    if num > mbz:
        return [generate_images_once(model, vq_model, args, seq, num=num, fill=lambda m, s, a: fill(m, [s], a)[0],
                                     decode=decode) for seq in seqs]
    per_group = mbz // num
    out = []
    model.eval()
    with torch.no_grad():
        for g0 in range(0, len(seqs), per_group):
            group = []
            for seq in seqs[g0:g0 + per_group]:
                seq = seq.clone()
                add_interlacing_beam_marks(seq, nb=num)
                group.append(seq)
            for rows in fill(model, group, args):
                out.append((rows, _decode_rows(rows, decode)))
    return out


def caption_ids(row, tokenizer=None):
    """The text ids after the last [ROI1] of a token row, un-offset as split_tokens gives them (what sentencepiece
    decodes)."""
    parts, _ = split_tokens(row.tolist() if torch.is_tensor(row) else row, tokenizer)
    idx = max(i for i, p in enumerate(parts) if p == '[ROI1]')
    return [x for p in parts[idx + 1:] if isinstance(p, list) for x in p]


def image2text(model, vq_model, args, images, num=8, fill=filling_shared_prompts, encode=None):
    """generate_samples.py:143-186, 202-221 for the 'image2text' task: `num` captions of every image.  images:
    [N, 3, 256, 256], normalised as vqvae.img2code takes them (the reference's read_img: Resize and CenterCrop 256,
    ToTensor, Normalize(IMG_MEAN, IMG_STD)).  The images are encoded (`encode`, default vqvae.img2code), each image's
    query is QUERY_TEMPLATES['image2text'] ([BASE] [BOI1] codes [EOI1] [ROI1] [MASK]*20) with beams marked as the
    reference marks them, nb = min(num, args.max_inference_batch_size), and whole images are packed into batches of at
    most args.max_inference_batch_size rows.  `fill` takes a list of templates and returns a list of token tensors:
    filling_shared_prompts reads each image's prompt K|V once for all of its beams, and falls back to
    filling_sequences where it does not apply.  Returns one (token rows [num, 1048], captions) pair per image; captions
    holds num lists of text ids (caption_ids: un-offset, for sentencepiece, which stays with the caller)."""
    encode = encode or (lambda imgs: vqvae.img2code(vq_model, imgs))
    tok = get_tokenizer(args)
    mbz = args.max_inference_batch_size
    assert num < mbz or num % mbz == 0
    nb = min(num, mbz)
    per_batch = max(1, mbz // nb)
    model.eval()
    with torch.no_grad():
        codes = encode(images)
        seqs = []
        for c in codes:
            seq = torch.tensor(build_query(QUERY_TEMPLATES['image2text'], [c.tolist()], tok), dtype=torch.long,
                               device=codes.device)
            add_interlacing_beam_marks(seq, nb=nb)
            seqs.append(seq)
        rows = [[] for _ in seqs]
        for g0 in range(0, len(seqs), per_batch):
            for _ in range(max(num // mbz, 1)):
                for i, r in enumerate(fill(model, [seq.clone() for seq in seqs[g0:g0 + per_batch]], args)):
                    rows[g0 + i].append(r)
    out = []
    for r in rows:
        r = torch.cat(r, dim=0)
        out.append((r, [caption_ids(row, tok) for row in r]))
    return out


def code_mask(pixel_mask):
    """A [N, 256, 256] pixel mask (True: regenerate) as the [N, 32, 32] mask of the codes of a 32 x 32 grid: a code is
    regenerated if any pixel of its 8 x 8 cell is masked."""
    n = pixel_mask.shape[0]
    assert tuple(pixel_mask.shape[1:]) == (256, 256), 'pixel masks are [N, 256, 256]'
    return pixel_mask.bool().view(n, 32, 8, 32, 8).any(dim=4).any(dim=2)


def completion_query(text, codes, mask, tokenizer=None):
    """The template that completes one image from its caption: [ROI1] text [BASE] [BOI1] codes, with -1 (generate) at
    every code where `mask` is True.  text: text ids (already offset into the unified vocabulary); codes: 1024 codes
    of a 32 x 32 grid in raster order; mask: [32, 32] or [1024] bool.  A mask of the codes after the first N gives
    build_query's '[ROI1] {} [BASE] [BOI1] [ImageN]{}' template.  Returns a list of ints."""
    codes = [int(x) for x in codes]
    mask = [bool(x) for x in torch.as_tensor(mask).reshape(-1).tolist()]
    assert len(codes) == len(mask) == 1024, 'completion works on 32 x 32 code grids'
    head = build_query('[ROI1] {} [BASE] [BOI1]', [text], tokenizer)
    return head + [-1 if m else c for c, m in zip(codes, mask)]


def complete_images(model, vq_model, args, texts, codes, masks, num=1, fill=filling_completions, decode=None):
    """The reference's "text and part of image" mode for many images: image i is completed from its caption texts[i]
    (text ids, already offset into the unified vocabulary) and the codes codes[i] ([N, 1024] int64, e.g.
    vqvae.img2code of the images) that masks[i] ([N, 32, 32] bool, True: regenerate; see code_mask) keeps.  Each
    image's template is completion_query's, with `num` beams marked as the reference marks them, nb = min(num,
    args.max_inference_batch_size), and whole images are packed into batches of at most args.max_inference_batch_size
    rows.  `fill` takes a list of templates and returns a list of token tensors: filling_completions runs the images of
    a batch as one ragged decode whatever their masks, and falls back to filling_sequence per template where it does
    not apply.  Every unmasked code is returned as given; the masked ones are drawn.  Returns one (token rows
    [num, len], images [num, 3, 256, 256]) pair per image, as generate_images_batch does."""
    decode = decode or (lambda c: vqvae.code2img(vq_model, c))
    tok = get_tokenizer(args)
    mbz = args.max_inference_batch_size
    assert num < mbz or num % mbz == 0
    assert len(texts) == codes.shape[0] == masks.shape[0], 'one text, code grid and mask per image'
    nb = min(num, mbz)
    per_batch = max(1, mbz // nb)
    seqs = []
    for text, c, m in zip(texts, codes, masks):
        seq = torch.tensor(completion_query(text, c, m, tok), dtype=torch.long, device=codes.device)
        add_interlacing_beam_marks(seq, nb=nb)
        seqs.append(seq)
    rows = [[] for _ in seqs]
    model.eval()
    with torch.no_grad():
        for g0 in range(0, len(seqs), per_batch):
            for _ in range(max(num // mbz, 1)):
                for i, r in enumerate(fill(model, [seq.clone() for seq in seqs[g0:g0 + per_batch]], args)):
                    rows[g0 + i].append(r)
        out = []
        for r in rows:
            r = torch.cat(r, dim=0)
            out.append((r, _decode_rows(r, decode)))
    return out


def super_resolution(model, vq_model, args, seq, fill=filling_sequence, decode=None, debug=False):
    """generate_samples.py:223-244: `seq` is the 'super-resolution' template filled in, [ROI1] text [BASE] [BOI1]
    followed by the 1024 codes of a 32 x 32 source image.  The source is magnified to 64 x 64 codes by `magnify`'s
    nine windows, and the grid is decoded by the VQ-VAE.  Returns (codes [1, 4096], images [n, 3, 512, 512]); n = 1,
    or 2 with debug=True, when the source image decoded and interpolated to 512 x 512 comes first, as the
    reference's debug output does."""
    decode = decode or (lambda codes: vqvae.code2img(vq_model, codes))
    tok = get_tokenizer(args)
    model.eval()
    with torch.no_grad():
        codes = magnify(model, tok, seq[-1024:], seq[:-1024], args, fill=fill)
        imgs = []
        if debug:
            src = decode(seq[-1024:].view(1, 32, 32))
            imgs.append(torch.nn.functional.interpolate(src, size=(512, 512)))
        imgs.append(decode(codes.view(1, 64, 64)))
    return codes, torch.cat(imgs, dim=0)


def super_resolution_batch(model, vq_model, args, seqs, fill=filling_sequences, decode=None):
    """super_resolution for many images: `seqs` is a list of filled 'super-resolution' templates, one per image (their
    text lengths may differ).  Images are magnified in groups of at most args.max_inference_batch_size by
    magnify_batch, whose `fill` runs each window of a group as one decode batch (filling_sequences: the given stretches
    of every window go through GPT2Model.chunk_run, the generated ones through the ragged decode graph); each
    magnified grid is then decoded by the VQ-VAE.  A group of one image, or a group whose templates cannot share a
    batch (filling_sequences falls back to filling_sequence per template, e.g. COGVIEW_B200_FAST_DECODE=0), gives
    what super_resolution gives.  Rows of a batch match solo runs within bf16 tolerance, not bit for bit (the abs-max
    LayerNorm scales are taken over the whole batch).  Returns (codes [N, 4096], images [N, 3, 512, 512])."""
    decode = decode or (lambda codes: vqvae.code2img(vq_model, codes))
    tok = get_tokenizer(args)
    mbz = max(1, args.max_inference_batch_size)
    codes = []
    model.eval()
    with torch.no_grad():
        for g0 in range(0, len(seqs), mbz):
            group = seqs[g0:g0 + mbz]
            if len(group) == 1:
                codes.append(magnify(model, tok, group[0][-1024:], group[0][:-1024], args,
                                     fill=lambda m, s, a, **kw: fill(m, [s], a)[0]))
                continue
            src = torch.stack([seq[-1024:] for seq in group])
            codes.append(magnify_batch(model, tok, src, [seq[:-1024] for seq in group], args, fill=fill))
        codes = torch.cat(codes, dim=0)
        imgs = torch.cat([decode(c.view(1, 64, 64)) for c in codes], dim=0)
    return codes, imgs


def post_selection_rows(rows, text, tokenizer=None):
    """The 'post-selection' query of every row `generate_images_once` returned: [BASE] [BOI1] codes [EOI1] [ROI1] text,
    where codes is the row's last image (the generated one) and `text` the caption's token ids (already offset into the
    unified vocabulary).  Returns a LongTensor [num, 2 + 1024 + 2 + len(text)] on the rows' device."""
    out = []
    for row in rows:
        _, images = split_tokens(row.tolist(), tokenizer)
        out.append(build_query(QUERY_TEMPLATES['post-selection'], [images[-1], text], tokenizer))
    return torch.tensor(out, dtype=torch.long, device=rows.device)


def post_selection(model, args, seq, score=inverse_prompt_score):
    """generate_samples.py:246-270 without the file output: `seq` holds one post-selection query per row ([num, len],
    see post_selection_rows); returns the caption log-likelihood of every row, scores [num], computed in groups of
    args.max_inference_batch_size rows.  The best candidates are scores.topk(k).indices."""
    num = seq.shape[0]
    mbz = args.max_inference_batch_size
    assert num < mbz or num % mbz == 0
    model.eval()
    with torch.no_grad():
        return torch.cat([score(model, seq[i * mbz:(i + 1) * mbz], args) for i in range(max(num // mbz, 1))], dim=0)


Reranked = namedtuple('Reranked', ['index', 'rows', 'images', 'scores', 'all_scores'])
Reranked.__doc__ = """The `keep` best of one caption's candidates, best first: index [keep] into its `num` draws, their
token rows [keep, len], images [keep, 3, H, W] and scores [keep], and the scores of all draws, all_scores [num].
index, scores and all_scores are on the CPU; rows and images stay where generation left them."""


def rerank(model, caption_model, vq_model, args, seqs, num, keep):
    """CogView's draw-many-keep-the-best recipe (generate_samples.py:147-200, 246-270) end to end, for many captions.
    seqs: 'text2image' templates, one per caption ([ROI1] caption [BASE] [BOI1] [MASK]*1024, 1-D LongTensors).
    `num` images per caption come from generate_images_batch with `model`; each is scored by `caption_model` (which may
    be `model` itself) as the log-likelihood of its caption given the image — the post-selection queries of all
    captions go through inverse_prompt_scores together, in groups of args.max_inference_batch_size rows.  Returns one
    Reranked per caption, holding its `keep` best candidates ordered by descending score, ties to the lower index."""
    assert 1 <= keep <= num
    tok = get_tokenizer(args)
    n_img = tok.img_tokenizer.num_tokens
    drawn = generate_images_batch(model, vq_model, args, seqs, num=num)
    queries = []
    for seq, (rows, _) in zip(seqs, drawn):
        text = [x + n_img for x in caption_ids(seq, tok)]
        queries.extend(post_selection_rows(rows, text, tok).unbind(0))
    caption_model.eval()
    scores = inverse_prompt_scores(caption_model, queries, args).cpu()
    out = []
    for c, (rows, imgs) in enumerate(drawn):
        s = scores[c * num:(c + 1) * num]
        index = torch.sort(s, descending=True, stable=True).indices[:keep]
        dev = index.to(rows.device)
        out.append(Reranked(index, rows[dev], imgs[index.to(imgs.device)], s[index], s))
    return out
