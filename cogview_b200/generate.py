"""Generation driver around `filling_sequence` — the token-level parts of generate_samples.py:68-200 and of
UnifiedTokenizer.parse_query / DecodeIds (data_utils/unified_tokenizer.py:91-196): query templates per task, query
assembly from already-tokenised text and image codes, beam batching, and decoding of the generated image codes
through the VQ-VAE.  Text <-> string conversion (sentencepiece) and image file I/O stay with the caller."""
import torch

from . import vqvae
from .generation.magnify import magnify
from .generation.sampling import add_interlacing_beam_marks, filling_sequence, get_tokenizer

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
        imgs = []
        for row in rows:
            _, images = split_tokens(row.tolist())
            codes = torch.tensor(images[-1], dtype=torch.long, device=rows.device).unsqueeze(0)
            img = decode(codes)
            if img.shape[-1] == 128:                       # low-level super-resolution sources are 128 x 128
                img = torch.nn.functional.interpolate(img, size=(256, 256))
            imgs.append(img)
    return rows, torch.cat(imgs, dim=0)


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
