"""Time sampling a list of captions: one caption after the other against all of them in one decode batch, 4B shape.

    python tools/caption_batch_time.py [--captions 16] [--images 4] [--gen 256] [--reps 2]

Seeded weights; caption c has 10 + 50 * c / (captions - 1) text tokens (10..60), in the text-to-image template
'[ROI1] text [BASE] [BOI1] [MASK]*gen' with `--images` beams.  Two routes, alternated in the same process:
  * loop  : filling_sequence once per caption (what generate_images_once runs per caption), `--images` rows per step;
  * batch : filling_sequences over all captions, captions x images rows per step (one ragged decode batch).
The VQ-VAE decode of the images is not part of either time.  Per route: total ms, ms per decode step (total over
`--gen` steps per caption, so it includes the prompts' forwards and the first draws), generated tokens/s; for the
batch route also the time of the per-caption prompt forwards alone, timed separately, and their share of the route.
Every shape is run once before it is timed and every window ends in a synchronise; the card's name and power limit
are printed with the numbers.  One JSON line per route.  Needs a GPU.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from decode_batch_time import card  # noqa: E402


def templates(n, images, gen):
    from cogview_b200.generation import sampling
    tok = sampling.get_tokenizer(bench.SampleArgs)
    g = torch.Generator().manual_seed(0)
    out = []
    for c in range(n):
        n_text = 10 + (50 * c) // max(1, n - 1)
        text = torch.randint(8192, 58192, (n_text,), generator=g).tolist()
        seq = [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + [-1] * gen
        sampling.add_interlacing_beam_marks(seq, nb=images)
        out.append(torch.tensor(seq, dtype=torch.long, device="cuda"))
    return out


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--captions", type=int, default=16)
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--gen", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("caption_batch_time: no GPU — a step time cannot be measured without one")
    from cogview_b200.generation import sampling

    class Args(bench.SampleArgs):
        max_inference_batch_size = a.captions * a.images
    cfg = bench.MODEL_4B
    torch.manual_seed(0)
    model = bench.build_model(cfg, cfg["max_sequence_length"], "cuda").eval()
    where = card()
    seqs = templates(a.captions, a.images, a.gen)

    def loop():
        for s in seqs:
            sampling.filling_sequence(model, s, Args)

    def batch():
        sampling.filling_sequences(model, seqs, Args)

    def prefills():
        for s in seqs:
            C = int((s >= 0).sum())
            tokens, mask, pos = sampling.get_batch(s[:C], s.device, Args)
            model(tokens, pos, mask, None, None, 0)

    routes = [("loop", loop, a.images), ("batch", batch, a.captions * a.images), ("prefills", prefills, 0)]
    for _, fn, _ in routes:                                    # warm every shape (graph capture, allocator, modules)
        timed(fn)
    ms = {name: [] for name, _, _ in routes}
    for _ in range(a.reps):                                    # alternate the routes
        for name, fn, _ in routes:
            ms[name].append(timed(fn))
    tokens = a.captions * a.images * a.gen
    for name, _, rows in routes[:2]:
        best = min(ms[name])
        steps = a.gen * (a.captions if name == "loop" else 1)
        rec = dict(route=name, captions=a.captions, images_per_caption=a.images, rows_per_step=rows,
                   gen_tokens=a.gen, ms=round(best, 2), ms_runs=[round(x, 2) for x in ms[name]],
                   ms_per_step=round(best / steps, 4), tokens_per_s=round(tokens / best * 1e3, 1), card=where)
        if name == "batch":
            rec["prefill_ms"] = round(min(ms["prefills"]), 2)
            rec["prefill_share"] = round(min(ms["prefills"]) / best, 4)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
