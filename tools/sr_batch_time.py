"""Time super-resolving many images: N calls of generate.super_resolution against one
generate.super_resolution_batch call, 4B shape, and the ragged chunk attention kernel on its own.

    python tools/sr_batch_time.py [--sizes 4,16,64] [--loop-images 4] [--reps 1]

Seeded weights (max_memory_length 1345); image i has its own 32 x 32 source codes and 20 + (3 * i) % 36 text tokens,
so the templates are 1047 tokens and longer; top-k 200, temperature 1.02 (DESIGN §5).  Routes, alternated in one
process after every shape has been run once:
  * loop  : super_resolution once per image.  One image's call does not depend on the others, so this route is timed
            over its first --loop-images images and reported per image;
  * batch : super_resolution_batch over N images (N rows per decode step; max_inference_batch_size = N).
The batch route's time is split into the per-window context prefills, the ragged chunk forwards (GPT2Model.chunk_run)
and the graph-replayed generate runs (each call wrapped in device synchronises, so the split sums to slightly less
than the whole).  Then cv_attn_chunk_ragged alone, CUDA events over 50 launches, at 17 tokens per row, 40 heads and
row lengths 1047 .. 1345 - 17: the cache bytes its rows' keys and values take, over its time.  The card's name and power
limit are read in the same run.  One JSON line per measurement.  Needs a GPU.
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


class SRArgs:
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
                              max_sequence_length=cfg["max_sequence_length"], max_memory_length=1345,
                              checkpoint_activations=False)
    finally:
        torch.set_default_dtype(old)
    return model.eval(), cfg


def templates(n):
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    tok = sampling.get_tokenizer(SRArgs)
    g = torch.Generator().manual_seed(2)
    out = []
    for i in range(n):
        text = torch.randint(8192, 58192, (20 + (3 * i) % 36,), generator=g).tolist()
        src = torch.randint(0, 8192, (1024,), generator=g).tolist()
        out.append(torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['super-resolution'], [text, src],
                                                     tokenizer=tok), dtype=torch.long, device="cuda"))
    return out


class Split:
    """Wraps the model's prefill forward, chunk_run and generate_run with synchronised host clocks."""

    def __init__(self, model):
        self.model = model
        self.ms = dict(prefill=0.0, chunk=0.0, graph=0.0)
        self.on = False
        for name, attr in (("chunk", "chunk_run"), ("graph", "generate_run")):
            setattr(model, attr, self._wrap(name, getattr(model, attr)))
        self.forward = model.forward
        model.forward = self._wrap("prefill", self.forward)

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


def time_kernel(cfg, where):
    from cogview_b200 import ops
    heads, h = cfg["num_attention_heads"], cfg["hidden_size"]
    n, max_len, cur_len = 17, 1345, 1345 - 17
    for b in (4, 16, 64):
        g = torch.Generator().manual_seed(b)
        pads = torch.randint(0, cur_len - 1047 + 1, (b,), generator=g).to(torch.int32)
        cache = torch.randn((b, max_len, 2 * h), device="cuda").to(torch.bfloat16)
        qkv = torch.randn((b, n, 3 * h), device="cuda").to(torch.bfloat16)
        pads_d = pads.cuda()
        nsplit = ops.attn_chunk_nsplit(b, heads, cur_len + n, qkv.device)
        for _ in range(5):
            ops.attn_chunk_ragged(qkv, cache, heads, cur_len, pads_d)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 50
        e0.record()
        for _ in range(reps):
            ops.attn_chunk_ragged(qkv, cache, heads, cur_len, pads_d)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        keys = int((cur_len - pads).sum()) + b * n
        cache_bytes = keys * 2 * h * 2                      # K and V of every key a row attends, bf16
        print(json.dumps(dict(measure="cv_attn_chunk_ragged", rows=b, tokens_per_row=n, heads=heads, nsplit=nsplit,
                              us=round(ms * 1e3, 2), cache_bytes=cache_bytes,
                              cache_GB_per_s=round(cache_bytes / (ms * 1e-3) / 1e9, 1), card=where)), flush=True)
        del cache, qkv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4,16,64")
    ap.add_argument("--loop-images", type=int, default=4)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--skip-routes", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sr_batch_time: no GPU — a time cannot be measured without one")
    from cogview_b200 import generate, vqvae
    where = card()
    print("card (name, power limit, max SM clock): %s" % where, flush=True)
    model, cfg = build_model()
    time_kernel(cfg, where)
    if a.skip_routes:
        return
    vq = vqvae.new_model()
    vq.load_state_dict(recipes.vqvae_state_dict(seed=0))
    vq = vq.cuda().eval()
    sizes = [int(x) for x in a.sizes.split(",")]
    seqs = templates(max(sizes + [a.loop_images]))
    split = Split(model)

    def loop():
        for s in seqs[:a.loop_images]:
            generate.super_resolution(model, vq, SRArgs, s)

    def batch(n):
        class A(SRArgs):
            max_inference_batch_size = n

        def run():
            codes, imgs = generate.super_resolution_batch(model, vq, A, seqs[:n])
            assert codes.shape == (n, 4096) and imgs.shape == (n, 3, 512, 512)
        return run

    routes = [("loop", loop, a.loop_images)] + [("batch", batch(n), n) for n in sizes]
    timed(routes[0][1] if a.loop_images <= 1 else (lambda: generate.super_resolution(model, vq, SRArgs, seqs[0])))
    for _, fn, _ in routes[1:]:                                  # warm every batch shape (graphs, caches, modules)
        timed(fn)
    res = {(name, n): [] for name, _, n in routes}
    splits = {}
    for _ in range(a.reps):                                      # alternate the routes
        for name, fn, n in routes:
            split.on = name == "batch"
            split.ms = dict(prefill=0.0, chunk=0.0, graph=0.0)
            res[(name, n)].append(timed(fn))
            splits[(name, n)] = dict(split.ms)
            split.on = False
    for name, _, n in routes:
        best = min(res[(name, n)])
        rec = dict(measure="super_resolution" if name == "loop" else "super_resolution_batch", images=n,
                   ms=round(best, 1), ms_runs=[round(x, 1) for x in res[(name, n)]],
                   s_per_image=round(best / n / 1e3, 3), images_per_s=round(n / best * 1e3, 4), card=where)
        if name == "batch":
            rec.update({k + "_ms": round(v, 1) for k, v in splits[(name, n)].items()})
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
