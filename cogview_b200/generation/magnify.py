"""Super-resolution driver (generation/magnify.py:22-43): a 32 x 32 code image is magnified to 64 x 64 by nine
overlapping windows; each window conditions on the text, its 16 x 16 source patch and the already generated rows
of its 32-column strip, and fills the rest through `filling_sequence` (`magnify`), or through `filling_sequences` for
many images at once (`magnify_batch`)."""
import math

import torch

from .sampling import filling_sequence, filling_sequences

# (window row, window column, number of 32-code lines generated or re-read in that window)
WINDOWS = [(0, 0, 18), (0, 1, 30), (0, 2, 30), (1, 1, 30), (1, 0, 30), (1, 2, 30), (2, 0, 32), (2, 1, 32), (2, 2, 32)]


def magnify(model, tokenizer, tokens_list, text_token_list, args, fill=filling_sequence):
    """tokens_list: [1024] codes of the 32 x 32 image; text_token_list: 1-D text prefix.  Returns [1, 4096] codes."""
    s = int(math.sqrt(len(tokens_list) + 1e-6))
    assert s == 32
    code = tokens_list.view(s, s)
    midfix = torch.tensor([tokenizer['[EOI1]'], tokenizer['[ROI2]'], tokenizer['[POS0]'], tokenizer['[BASE]'],
                           tokenizer['[BOI2]']], device=code.device)
    magnified = code.new_zeros((s * 2, s * 2), dtype=torch.long) - 1
    for i, j, line in WINDOWS:
        code_part = code[8 * i: 8 * (i + 2), 8 * j: 8 * (j + 2)].reshape(-1)
        known = magnified[16 * i: 16 * i + line, 16 * j: 16 * (j + 2)].reshape(-1)      # -1 = still to generate
        context = torch.cat([text_token_list, code_part, midfix], dim=0)
        seq = torch.cat([context, known], dim=0)
        done = fill(model, seq, args, invalid_slices=[slice(tokenizer.img_tokenizer.num_tokens, None)])
        magnified[16 * i: 16 * i + line, 16 * j: 16 * (j + 2)] = done[0, len(context):].view(line, 32)
    return magnified.view(1, s * s * 4)


def magnify_batch(model, tokenizer, codes, texts, args, fill=filling_sequences):
    """magnify for N images at once: codes [N, 1024] (one 32 x 32 code image per row), texts: N 1-D text prefixes
    (their lengths may differ).  The nine windows are walked once; each window's template is built per image from that
    image's own magnified grid, exactly as magnify builds it, and the N templates are filled by one `fill` call
    (a list of templates -> a list of [1, len] token tensors, see filling_sequences).  Returns [N, 4096] codes."""
    n = codes.shape[0]
    assert codes.shape[1] == 1024 and len(texts) == n
    s = 32
    code = codes.view(n, s, s)
    midfix = torch.tensor([tokenizer['[EOI1]'], tokenizer['[ROI2]'], tokenizer['[POS0]'], tokenizer['[BASE]'],
                           tokenizer['[BOI2]']], device=code.device)
    magnified = code.new_zeros((n, s * 2, s * 2), dtype=torch.long) - 1
    for i, j, line in WINDOWS:
        seqs, ctx_len = [], []
        for r in range(n):
            code_part = code[r, 8 * i: 8 * (i + 2), 8 * j: 8 * (j + 2)].reshape(-1)
            known = magnified[r, 16 * i: 16 * i + line, 16 * j: 16 * (j + 2)].reshape(-1)
            context = torch.cat([texts[r], code_part, midfix], dim=0)
            seqs.append(torch.cat([context, known], dim=0))
            ctx_len.append(len(context))
        done = fill(model, seqs, args)
        for r in range(n):
            magnified[r, 16 * i: 16 * i + line, 16 * j: 16 * (j + 2)] = done[r][0, ctx_len[r]:].view(line, 32)
    return magnified.view(n, s * s * 4)
