"""Cost of nucleus (top-p) sampling on the H100: the fused sampling kernel alone, and the 4B decode step end to end.

    python tools/top_p_time.py [--batches 1,8,16,64] [--launches 200] [--e2e 4,16,64] [--gen 512] [--reps 2]

Kernel: cv_sample_topk at top_p 0.9 and at top_p 0 on the same fp32 [b, 58240] logits (randn x 3), over the
8192 image codes and over the text range, top_k 0 and 200; each timed with CUDA events over `--launches` launches,
the two alternated three times, the fastest window kept.  End to end: filling_sequence on the 4B shape (seeded
weights, bench.py's 65-token text2image context) with `--gen` generated tokens per sequence at nb beams, top_k 200,
top_p 0.9 against top_p 0, alternated in one process; ms per generated step of the whole run (the context forward
and the first, host-drawn slot included).  Every shape is run once before it is timed and every window ends in a
synchronise.  The card's name, power limit and max SM clock are read in the same run and printed with the numbers.
One JSON line per measurement.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402

V = 58240
RANGES = {"image": [(0, 8192)], "text": [(8192, 58192)]}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return "%s (%s)" % (name, q)


def time_kernel(logits, top_k, valid, top_p, launches):
    from cogview_b200 import ops
    ids = torch.empty(logits.shape[0], dtype=torch.int64, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(launches):
        ops.sample_topk(logits, 1.0, top_k, valid, seed=i, next_ids=ids, top_p=top_p)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def kernels(batches, launches, where):
    for b in batches:
        logits = (torch.randn((b, V), device="cuda", generator=torch.Generator(device="cuda").manual_seed(b)) * 3.0)
        for rname, valid in RANGES.items():
            for top_k in (0, 200):
                us = {0.0: [], 0.9: []}
                for top_p in us:                                # warm-up
                    time_kernel(logits, top_k, valid, top_p, 5)
                for _ in range(3):
                    for top_p in us:
                        us[top_p].append(time_kernel(logits, top_k, valid, top_p, launches))
                print(json.dumps(dict(what="kernel", b=b, valid=rname, top_k=top_k, launches=launches,
                                      us_topk=round(min(us[0.0]), 2), us_topk_topp=round(min(us[0.9]), 2),
                                      us_runs_topk=[round(x, 2) for x in us[0.0]],
                                      us_runs_topk_topp=[round(x, 2) for x in us[0.9]], card=where)), flush=True)


def end_to_end(model, batches, gen, reps, where):
    from cogview_b200.generation import sampling

    class Plain(bench.SampleArgs):
        top_k, top_p = 200, 0.0

    class Nucleus(Plain):
        top_p = 0.9
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run(seq, args):
        with torch.no_grad():
            e0.record()
            sampling.filling_sequence(model, seq, args)
            e1.record()
            torch.cuda.synchronize()
        return e0.elapsed_time(e1) / gen

    for nb in batches:
        seq = bench.make_template(nb, gen, seed=0).cuda()
        ms = {"top_p=0": [], "top_p=0.9": []}
        modes = (("top_p=0", Plain), ("top_p=0.9", Nucleus))
        for _, args in modes:                                  # warm-up: graph capture, allocator
            run(seq, args)
        for _ in range(reps):
            for name, args in modes:
                ms[name].append(run(seq, args))
        print(json.dumps(dict(what="filling_sequence", model="4B", nb=nb, gen_tokens=gen, top_k=200,
                              ms_per_step_top_p0=round(min(ms["top_p=0"]), 4),
                              ms_per_step_top_p09=round(min(ms["top_p=0.9"]), 4),
                              runs={k: [round(x, 4) for x in v] for k, v in ms.items()}, card=where)), flush=True)
        model.transformer._kv_pool = {}
        model.transformer._kv = None
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,16,64")
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--e2e", default="4,16,64")
    ap.add_argument("--gen", type=int, default=512)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("top_p_time: no GPU — kernel and step times cannot be measured without one")
    where = card()
    print(json.dumps(dict(card=where)), flush=True)
    kernels([int(x) for x in a.batches.split(",")], a.launches, where)
    if a.e2e:
        cfg = bench.MODEL_4B
        torch.manual_seed(0)
        model = bench.build_model(cfg, cfg["max_sequence_length"], "cuda").eval()
        end_to_end(model, [int(x) for x in a.e2e.split(",")], a.gen, a.reps, where)


if __name__ == "__main__":
    main()
