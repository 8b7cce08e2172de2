"""Measurements that are claimed in DESIGN.md but are not part of bench.py's headline line:

  sweep     : SURVEY §8(d) config 2 batch sweep — AR sampling tokens/s of the 4B model at b = 1, 4, 8 (persistent
              one-kernel step), 16 (per-operation decode kernels, cv_linear_small_m M <= 16) and 64 (general wgmma
              GEMM path with the K|V cache)
  sr_dense  : BASELINE configs[4] as the reference SHIPS it (scripts/super_resolution.sh:7,36): dense attention,
              1345 positions — context 321 tokens, 1024 generated, 4 beams
  sr_sparse : BASELINE configs[4] as the config names it: is_sparse = 2 (sparse_attention_inference,
              mpu/sparse_transformer.py:498-520,591-600,727-750), 4096 positions, query_window 128 x 6, 768 pivots;
              fresh Python random.sample pivots per layer per token as in the reference (host-bound by construction)

    python tools/bench_extra.py [sweep] [sr_dense] [sr_sparse] [--gen 1024]

One JSON line per measurement (CUDA events around whole filling_sequence calls, 1 warm-up + 2 timed)."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402


def timed_fill(model, seq, args_obj, reps=2):
    from cogview_b200.generation import sampling
    with torch.no_grad():
        sampling.filling_sequence(model, seq, args_obj)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            out = sampling.filling_sequence(model, seq, args_obj)
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", nargs="*", default=["sweep", "sr_dense", "sr_sparse"])
    ap.add_argument("--gen", type=int, default=1024)
    ap.add_argument("--gen-sparse", type=int, default=2048)
    ap.add_argument("--batches", default="1,4,8,16,64")
    a = ap.parse_args()
    from cogview_b200.generation import sampling
    out_lines = []
    if "sweep" in a.what:
        cfg = bench.MODEL_4B
        model = bench.build_model(cfg, cfg["max_sequence_length"], "cuda").eval()
        for b in [int(x) for x in a.batches.split(",")]:
            seq = bench.make_template(b, a.gen, seed=0).cuda()
            ms, out = timed_fill(model, seq, bench.SampleArgs)
            path = "persistent one-kernel step" if b <= 8 else ("per-operation decode kernels" if b <= 16
                                                                else "general GEMM path + K|V cache")
            out_lines.append(dict(workload="batch sweep", batch=b, gen_tokens=a.gen, ms=ms, tokens_per_s=b * a.gen / ms * 1e3,
                                  ms_per_token_step=ms / a.gen, path=path))
            print(json.dumps(out_lines[-1]), flush=True)
            model.transformer._kv_pool = {}
            torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    if "sr_dense" in a.what:
        cfg = dict(bench.MODEL_4B, max_sequence_length=1345)
        model = bench.build_model(cfg, 1345, "cuda").eval()
        tok = sampling.get_tokenizer(bench.SampleArgs)
        g = torch.Generator().manual_seed(1)
        text = torch.randint(8192, 58192, (62,), generator=g).tolist()
        low = torch.randint(0, 8192, (256,), generator=g).tolist()
        seq = [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + low + [-1] * (1345 - 321)
        sampling.add_interlacing_beam_marks(seq, nb=4)
        seq = torch.tensor(seq, dtype=torch.long).cuda()
        ms, out = timed_fill(model, seq, bench.SampleArgs)
        n = 1345 - 321
        out_lines.append(dict(workload="configs[4] dense SR shape (1345 positions, is_sparse=0)", batch=4, gen_tokens=n, ms=ms,
                              tokens_per_s=4 * n / ms * 1e3, ms_per_token_step=ms / n))
        print(json.dumps(out_lines[-1]), flush=True)
        del model
        torch.cuda.empty_cache()
    if "sr_sparse" in a.what:
        cfg = dict(bench.MODEL_4B, max_sequence_length=4096)
        model = bench.build_model(cfg, 4096, "cuda").eval()

        class SparseArgs(bench.SampleArgs):
            is_sparse = 2
        import random
        random.seed(1234)
        tok = sampling.get_tokenizer(SparseArgs)
        g = torch.Generator().manual_seed(2)
        text = torch.randint(8192, 58192, (62,), generator=g).tolist()
        low = torch.randint(0, 8192, (256,), generator=g).tolist()
        for pivots, n in (("device", min(a.gen_sparse, 4096 - 322)), ("host", min(256, a.gen_sparse))):
            os.environ["COGVIEW_B200_SPARSE_PIVOTS"] = pivots
            seq = [tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + low + [-1] * n
            sampling.add_interlacing_beam_marks(seq, nb=4)
            seq = torch.tensor(seq, dtype=torch.long).cuda()
            ms, out = timed_fill(model, seq, SparseArgs, reps=1)
            out_lines.append(dict(
                workload="configs[4] sparse generation (4096 positions, is_sparse=2, window 128x6, 768 pivots), 321-token context",
                pivots=pivots, batch=4, gen_tokens=n, ms=ms, tokens_per_s=4 * n / ms * 1e3, ms_per_token_step=ms / n,
                note=("key lists of all layers from one cv_sparse_plan launch per token, gathered attention, CUDA graph"
                      if pivots == "device" else
                      "fresh random.sample pivots per layer per token on the host, as the reference does")))
            print(json.dumps(out_lines[-1]), flush=True)
    os.makedirs(os.path.join(bench.ROOT, "gpurun_out"), exist_ok=True)
    json.dump(out_lines, open(os.path.join(bench.ROOT, "gpurun_out", "bench_extra.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
