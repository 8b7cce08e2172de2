"""Time captioning images (image2text) three ways at the 4B shape, and the shared-prefix decode attention on its own.

    python tools/image2text_time.py [--images 8] [--num 8] [--reps 2] [--skip-routes]

Seeded weights (max_memory_length 1089, as scripts/image2text.sh's --max-position-embeddings), seeded VQ-VAE, seeded
256 x 256 images; 8 beams per image, top-k 200, temperature 1.0.  Every route is generate.image2text with another
`fill`, so each also encodes the images; the routes are alternated in one process after each has run once:
  * once   : filling_sequence per image (what the reference runs for each image): a batch-1 prompt forward, then
             num rows per decode step;
  * ragged : filling_sequences over all images: a batch-1 prompt forward per image, its K|V copied into its num rows of
             one images x num-row cache, then one ragged decode run;
  * shared : filling_shared_prompts (the default): one prompt forward at batch `images`, then one decode run in which
             each image's prompt K|V is read once for all of its beams (cv_attn_decode_shared).
Per route: total ms, s per image, and the prompt forwards and the decode runs, each call timed between device
synchronises (so the split sums to a little less than the total): prompt-forward ms and decode ms per step.  Then
cv_attn_decode_shared against cv_attn_decode with row_pad on copied prefixes (8 groups x 8 rows, 40 heads, P = 1028,
s = 10), CUDA events over 200 launches each: the K|V bytes each kernel must read and GB/s against 3350 GB/s.  The
card's name and power limit are read in the same run.  One JSON line per measurement.  Needs a GPU.
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

HBM_GBPS = 3350.0          # H100 SXM data sheet


class CapArgs:
    temperature = 1.0
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
    return model.eval(), cfg


def images(n):
    from cogview_b200.vqvae.api import IMG_MEAN, IMG_STD
    img = torch.rand((n, 3, 256, 256), generator=torch.Generator().manual_seed(1))
    return ((img - torch.tensor(IMG_MEAN).view(1, 3, 1, 1)) / torch.tensor(IMG_STD).view(1, 3, 1, 1)).cuda()


class Split:
    """Times the model's prompt forwards and decode runs (generate_run, shared_run) with synchronised host clocks."""

    def __init__(self, model):
        self.ms = dict(prompt=0.0, decode=0.0)
        self.steps = 0
        self.on = False
        model.forward = self._wrap("prompt", model.forward)
        for attr in ("generate_run", "shared_run"):
            setattr(model, attr, self._wrap("decode", getattr(model, attr)))

    def _wrap(self, name, fn):
        def run(*a, **kw):
            if not self.on:
                return fn(*a, **kw)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **kw)
            torch.cuda.synchronize()
            self.ms[name] += (time.perf_counter() - t0) * 1e3
            if name == "decode":
                self.steps += a[3]                        # n_steps of generate_run / shared_run
            return r
        return run


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def time_kernels(cfg, where, groups=8, G=8, P=1028, s=10, reps=200):
    from cogview_b200 import ops
    heads, h = cfg["num_attention_heads"], cfg["hidden_size"]
    b, s_max, max_len = groups * G, 20, 1089
    prefix = torch.randn((groups, max_len, 2 * h), device="cuda").to(torch.bfloat16)
    suffix = torch.randn((b, s_max, 2 * h), device="cuda").to(torch.bfloat16)
    cache = torch.empty((b, max_len, 2 * h), dtype=torch.bfloat16, device="cuda")
    for r in range(b):                                    # the same keys, one copy of the prompt per row
        cache[r, :P] = prefix[r // G, :P]
        cache[r, P:P + s] = suffix[r, :s]
    qkv = torch.randn((b, 3 * h), device="cuda").to(torch.bfloat16)
    s_dev = torch.tensor([s], dtype=torch.int32, device="cuda")
    cur = torch.tensor([P + s], dtype=torch.int32, device="cuda")
    pads = torch.zeros(b, dtype=torch.int32, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nsplit_ragged = max(1, min(16, -(-8 * sms // (b * heads))))           # what DecodeRunner picks
    nsplit_shared = ops.attn_chunk_nsplit(groups, heads, P, qkv.device)
    out_s = ops.attn_decode_shared(qkv, prefix, suffix, heads, P, s_dev=s_dev, nsplit=nsplit_shared)
    out_r = ops.attn_decode(qkv, cache, heads, cur_len_dev=cur, nsplit=nsplit_ragged, row_pad=pads)
    err = (out_s.float() - out_r.float()).abs().max().item()
    runs = dict(
        cv_attn_decode_shared=(lambda: ops.attn_decode_shared(qkv, prefix, suffix, heads, P, s_dev=s_dev,
                                                              nsplit=nsplit_shared),
                               (groups * P + b * (s + 1)) * 2 * h * 2, nsplit_shared),
        cv_attn_decode=(lambda: ops.attn_decode(qkv, cache, heads, cur_len_dev=cur, nsplit=nsplit_ragged,
                                                row_pad=pads),
                        b * (P + s + 1) * 2 * h * 2, nsplit_ragged))
    for name, (fn, nbytes, nsplit) in runs.items():
        for _ in range(10):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        gbps = nbytes / (ms * 1e-3) / 1e9
        print(json.dumps(dict(measure=name, groups=groups, rows=b, heads=heads, P=P, s=s, nsplit=nsplit,
                              us=round(ms * 1e3, 2), kv_bytes=nbytes, GB_per_s=round(gbps, 1),
                              share_of_3350=round(gbps / HBM_GBPS, 3), max_abs_diff_vs_other=err, card=where)),
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--num", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--skip-routes", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("image2text_time: no GPU — a time cannot be measured without one")
    from cogview_b200 import generate, vqvae
    from cogview_b200.generation import sampling
    where = card()
    print("card (name, power limit, max SM clock): %s" % where, flush=True)
    model, cfg = build_model()
    time_kernels(cfg, where)
    if a.skip_routes:
        return
    vq = vqvae.new_model()
    vq.load_state_dict(recipes.vqvae_state_dict(seed=0))
    vq = vq.cuda().eval()
    imgs = images(a.images)
    split = Split(model)
    fills = [("once", lambda m, seqs, args: [sampling.filling_sequence(m, s, args) for s in seqs]),
             ("ragged", sampling.filling_sequences),
             ("shared", sampling.filling_shared_prompts)]

    def route(fill):
        def run():
            out = generate.image2text(model, vq, CapArgs, imgs, num=a.num, fill=fill)
            assert len(out) == a.images and all(r.shape == (a.num, 1048) for r, _ in out)
        return run
    for _, fill in fills:                                        # warm every route (graphs, caches, modules)
        timed(route(fill))
    res = {name: [] for name, _ in fills}
    splits = {}
    for _ in range(a.reps):
        for name, fill in fills:
            split.on = True
            split.ms, split.steps = dict(prompt=0.0, decode=0.0), 0
            res[name].append(timed(route(fill)))
            splits[name] = (dict(split.ms), split.steps)
            split.on = False
    for name, _ in fills:
        best = min(res[name])
        ms, steps = splits[name]
        print(json.dumps(dict(measure="image2text", route=name, images=a.images, beams=a.num, ms=round(best, 1),
                              ms_runs=[round(x, 1) for x in res[name]], s_per_image=round(best / a.images / 1e3, 4),
                              prompt_forward_ms=round(ms["prompt"], 1), decode_ms=round(ms["decode"], 1),
                              decode_steps=steps, decode_ms_per_step=round(ms["decode"] / max(steps, 1), 2),
                              card=where)), flush=True)


if __name__ == "__main__":
    main()
