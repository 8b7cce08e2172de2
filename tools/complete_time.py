"""Time completing partly given images: generate.complete_images with filling_completions (all images of a batch in one
ragged decode) against the per-template loop (filling_sequence once per image), 4B shape.

    python tools/complete_time.py [--sizes 16,64] [--loop-images 4] [--reps 2]

Seeded weights (max_memory_length 1089); image i has its own 32 x 32 codes, 20 + (3 * i) % 36 text tokens and its own
random rectangle of 4 .. 16 x 4 .. 16 codes to regenerate; one completion per image; top-k 200, temperature 1.02.
Routes, alternated in one process after every shape has been run once:
  * loop  : complete_images whose fill runs filling_sequence per template (each given stretch a multi-token forward,
            each generated stretch a graph-replayed run at batch 1).  One image does not depend on the others, so this
            route is timed over its first --loop-images images and reported per image;
  * batch : complete_images over N images with max_inference_batch_size = N (N rows per decode step).
Both include the VQ-VAE decode of the images.  The batch route's time is split into the per-image prefills and the one
graph-replayed decode of S steps (each call wrapped in device synchronises, so the split sums to slightly less than
the whole); S, the number of decode steps, is reported with it.  The card's name, power limit and maximum SM clock are
read in the same run.  One JSON line per measurement.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import recipes  # noqa: E402


class CArgs:
    temperature = 1.02
    top_k = 200
    top_p = 0.0
    is_sparse = 0
    img_tokenizer_num_tokens = 8192
    max_inference_batch_size = 64


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def build_model():
    from cogview_b200.model import GPT2Model
    cfg = dict(recipes.COGVIEW_4B)
    torch.manual_seed(0)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            model = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"],
                              hidden_size=cfg["hidden_size"], num_attention_heads=cfg["num_attention_heads"],
                              embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                              max_sequence_length=cfg["max_sequence_length"], max_memory_length=1089,
                              checkpoint_activations=False)
    finally:
        torch.set_default_dtype(old)
    model.transformer.mems_mode = "kv"
    return model.eval(), cfg


def inputs(n):
    g = torch.Generator().manual_seed(2)
    texts, codes, masks = [], [], []
    for i in range(n):
        texts.append(torch.randint(8192, 58192, (20 + (3 * i) % 36,), generator=g).tolist())
        codes.append(torch.randint(0, 8192, (1024,), generator=g))
        h, w = (int(x) for x in torch.randint(4, 17, (2,), generator=g))
        i0, j0 = int(torch.randint(0, 33 - h, (1,), generator=g)), int(torch.randint(0, 33 - w, (1,), generator=g))
        m = torch.zeros((32, 32), dtype=torch.bool)
        m[i0:i0 + h, j0:j0 + w] = True
        masks.append(m)
    return texts, torch.stack(codes).cuda(), torch.stack(masks).cuda()


class Split:
    """Wraps the model's prefill forward and generate_run with synchronised host clocks."""

    def __init__(self, model):
        self.ms = dict(prefill=0.0, decode=0.0)
        self.on = False
        model.generate_run = self._wrap("decode", model.generate_run)
        model.forward = self._wrap("prefill", model.forward)

    def _wrap(self, name, fn):
        def run(*a, **kw):
            if not self.on:
                return fn(*a, **kw)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **kw)
            torch.cuda.synchronize()
            self.ms[name] += (time.perf_counter() - t0) * 1e3
            return r
        return run


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,64")
    ap.add_argument("--loop-images", type=int, default=4)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("complete_time: no GPU — a time cannot be measured without one")
    from cogview_b200 import generate, vqvae
    from cogview_b200.generation import sampling
    where = card()
    print("card (name, power limit, max SM clock): %s" % where, flush=True)
    model, cfg = build_model()
    vq = vqvae.new_model()
    vq.load_state_dict(recipes.vqvae_state_dict(seed=0))
    vq = vq.cuda().eval()
    sizes = [int(x) for x in a.sizes.split(",")]
    texts, codes, masks = inputs(max(sizes + [a.loop_images]))
    tok = sampling.get_tokenizer(CArgs)
    split = Split(model)

    def per_template(m, seqs, args):
        return [sampling.filling_sequence(m, s, args) for s in seqs]

    def run(n, fill):
        class A(CArgs):
            max_inference_batch_size = n

        def go():
            out = generate.complete_images(model, vq, A, texts[:n], codes[:n], masks[:n], num=1, fill=fill)
            assert len(out) == n and out[0][1].shape == (1, 3, 256, 256)
        return go

    steps = {}
    for n in sizes:
        tmpls = [generate.completion_query(t, c, m, tok) for t, c, m in zip(texts[:n], codes[:n], masks[:n])]
        with torch.no_grad():
            _, S, ok = sampling._completion_plan(model, tmpls, CArgs, tok)
        assert ok, "the batch route does not apply to %d images" % n
        steps[n] = S
    routes = [("loop", run(a.loop_images, per_template), a.loop_images)] + [
        ("batch", run(n, sampling.filling_completions), n) for n in sizes]
    for _, fn, _ in routes:                                       # warm every shape (graphs, caches, modules)
        timed(fn)
    res = {(name, n): [] for name, _, n in routes}
    splits = {}
    for _ in range(a.reps):                                      # alternate the routes
        for name, fn, n in routes:
            split.on = name == "batch"
            split.ms = dict(prefill=0.0, decode=0.0)
            res[(name, n)].append(timed(fn))
            splits[(name, n)] = dict(split.ms)
            split.on = False
    for name, _, n in routes:
        best = min(res[(name, n)])
        rec = dict(measure="complete_images " + name, images=n, ms=round(best, 1),
                   ms_runs=[round(x, 1) for x in res[(name, n)]], s_per_image=round(best / n / 1e3, 3),
                   images_per_s=round(n / best * 1e3, 3), card=where)
        if name == "batch":
            rec.update(steps=steps[n], **{k + "_ms": round(v, 1) for k, v in splits[(name, n)].items()})
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
