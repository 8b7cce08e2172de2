"""Time per decode step against the number of sequences sampled together (SURVEY §8(d) config 2 batch sweep), 4B shape.

    python tools/decode_batch_time.py [--batches 4,16,32,64] [--gen 1024] [--gen-general 128] [--reps 2]

Seeded weights, a 64-token context ([ROI1] + 62 text tokens + [BASE] [BOI1] is 65; the first image token comes from
the context's forward), `--gen` generated tokens per sequence through filling_sequence.  Per batch size: ms per
step, tokens/s, and the bf16 weight bytes every step has to read over the step time, next to the H100 SXM data-sheet
HBM rate (3.35 TB/s) — an end-to-end rate of the whole step (attention, LayerNorms, sampling and launch gaps
included), not a kernel's share of peak.

Above 16 sequences the general route (COGVIEW_B200_FAST_DECODE=0: training GEMM tiles, cv_attn_fwd with one query,
sampling on the host) is timed as well, alternating with the graph route in the same process, with `--gen-general`
tokens (it pays host work per token; the count is printed with the number).  Every timed shape is run once before
it is timed, every window ends in a synchronise; the card's name and power limit are printed with the numbers.
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

HBM_PEAK_GBS = 3350.0


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return "%s (%s)" % (name, q)


def timed_fill(model, seq, reps):
    from cogview_b200.generation import sampling
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        e0.record()
        for _ in range(reps):
            sampling.filling_sequence(model, seq, bench.SampleArgs)
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="4,16,32,64")
    ap.add_argument("--gen", type=int, default=1024)
    ap.add_argument("--gen-general", type=int, default=128)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("decode_batch_time: no GPU — a step time cannot be measured without one")
    from cogview_b200 import ops
    cfg = bench.MODEL_4B
    torch.manual_seed(0)
    model = bench.build_model(cfg, cfg["max_sequence_length"], "cuda").eval()
    weight_bytes = 2 * bench.param_count(model)
    where = card()
    for b in [int(x) for x in a.batches.split(",")]:
        routes = [("graph", "1", a.gen)]
        if b > ops.DECODE_SMALL_MAX_BATCH:
            routes.append(("general", "0", a.gen_general))
        seqs = {name: bench.make_template(b, gen, seed=0).cuda() for name, _, gen in routes}
        for name, env, _ in routes:                             # warm every shape (graph capture, allocator, modules)
            os.environ["COGVIEW_B200_FAST_DECODE"] = env
            timed_fill(model, seqs[name], 1)
        ms = {name: [] for name, _, _ in routes}
        for _ in range(a.reps):                                 # alternate the routes
            for name, env, _ in routes:
                os.environ["COGVIEW_B200_FAST_DECODE"] = env
                ms[name].append(timed_fill(model, seqs[name], 1))
        for name, _, gen in routes:
            step = min(ms[name]) / gen
            print(json.dumps(dict(batch=b, route=name, gen_tokens=gen, ms_per_step=round(step, 4),
                                  ms_per_step_runs=[round(x / gen, 4) for x in ms[name]],
                                  tokens_per_s=round(b / step * 1e3, 1),
                                  weight_gb_per_s=round(weight_bytes / step / 1e6, 1), hbm_data_sheet_gb_per_s=HBM_PEAK_GBS,
                                  weight_bytes=weight_bytes, card=where)), flush=True)
        os.environ["COGVIEW_B200_FAST_DECODE"] = "1"
        model.transformer._kv_pool = {}
        model.transformer._kv = None
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
