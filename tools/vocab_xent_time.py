"""Time the fused vocabulary cross-entropy (GPT2Model.forward(..., labels=)) against the logits route.

    python tools/vocab_xent_time.py [--parts stage,step,fit] [--reps 5] [--max-seqs 64]

  stage : the loss stage alone at K = 2560, V = 58240, M = 2176 and 8704 rows: forward + backward of
          _LogitsFn + mpu.vocab_parallel_cross_entropy ("old") and of _VocabXentFn ("new"), alternated in one process.
          Time per call (median of --reps, CUDA events) and the rise of torch.cuda.max_memory_allocated over a call.
          Then cv_vocab_xent_dlogits alone over the whole vocabulary (CUDA events over 10 launches): TFLOP/s of its
          2 M K V operations.
  step  : pretrain.train_step with FusedAdamW on the 4B shape (seeded random weights) at 2 x 1088 tokens without
          activation recompute, fused_loss False and True alternated: step time (median, host clock around
          synchronised steps) and torch.cuda.max_memory_allocated.
  fit   : with checkpoint_activations=True, the largest number of 1088-token sequences per step that runs on each
          route (doubling, then bisection; a size fits when reps + 1 consecutive steps run without running out of
          memory), and tokens/s at that size (median of those steps but the first).
The card's name, power limit and maximum SM clock are read in the same run.  One JSON line per measurement.
Needs a GPU.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import recipes  # noqa: E402

V = 58240
K4B = 2560


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def emit(**kw):
    print(json.dumps(kw), flush=True)


def events_ms(fn, reps):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def part_stage(reps):
    from cogview_b200 import mpu, ops
    from cogview_b200.model.gpt2_modeling import _LogitsFn, _VocabXentFn
    g = torch.Generator(device="cuda").manual_seed(0)
    w = (torch.randn((V, K4B), generator=g, device="cuda") * 0.02).to(torch.bfloat16).requires_grad_(True)
    for M in (2176, 8704):
        h = torch.randn((M, K4B), generator=g, device="cuda").to(torch.bfloat16).requires_grad_(True)
        t = torch.randint(0, V, (M,), generator=g, device="cuda")

        def old():
            losses = mpu.vocab_parallel_cross_entropy(_LogitsFn.apply(h, w).float(), t)
            losses.mean().backward()

        def new():
            losses = _VocabXentFn.apply(h, w, t, None)
            losses.mean().backward()

        res = {"old": [], "new": []}
        peak = {}
        for name, fn in (("old", old), ("new", new)):     # warm-up
            h.grad = w.grad = None
            fn()
        for _ in range(reps):
            for name, fn in (("old", old), ("new", new)):
                h.grad = w.grad = None
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                res[name].append(events_ms(fn, 1))
                peak[name] = torch.cuda.max_memory_allocated() - base
        for name in ("old", "new"):
            emit(part="stage", route=name, M=M, K=K4B, V=V, ms=round(statistics.median(res[name]), 3),
                 peak_rise_mb=round(peak[name] / 1e6, 1), chunks=len(ops.xent_chunks(M, V)) if name == "new" else None)
        with torch.no_grad():
            _, lse = ops.vocab_xent_fwd(h.detach(), w.detach(), t)
            gl = torch.full((M,), 1.0 / M, device="cuda")
            d = torch.empty((M, V), dtype=torch.bfloat16, device="cuda")

            def dl():
                for _ in range(10):
                    ops.vocab_xent_dlogits(h.detach(), w.detach(), t, lse, gl, 0, V, out=d)
            dl()
            ms = events_ms(dl, 3) / 10
            emit(part="dlogits_kernel", M=M, K=K4B, V=V, us=round(ms * 1e3, 1),
                 tflops=round(2.0 * M * K4B * V / (ms / 1e3) / 1e12, 1))
            del d
        h.grad = w.grad = None
        del h
        gc.collect()
        torch.cuda.empty_cache()
    del w


def build_4b(ckpt):
    from cogview_b200.model import GPT2Model, gpt2_get_params_for_weight_decay_optimization
    from cogview_b200.optim import FusedAdamW
    cfg = recipes.COGVIEW_4B
    torch.manual_seed(0)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            model = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"],
                              hidden_size=cfg["hidden_size"], num_attention_heads=cfg["num_attention_heads"],
                              embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                              max_sequence_length=cfg["max_sequence_length"], max_memory_length=0,
                              checkpoint_activations=ckpt)
    finally:
        torch.set_default_dtype(old)
    groups = gpt2_get_params_for_weight_decay_optimization(model)
    opt = FusedAdamW(groups, lr=1e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_grad_norm=1.0)
    return model.train(), opt


def make_batch(b, seed):
    from cogview_b200.generation.sampling import get_masks_and_position_ids
    s = recipes.COGVIEW_4B["max_sequence_length"] - 1
    g = torch.Generator().manual_seed(seed)
    tok = torch.cat((torch.randint(8192, 58192, (b, 64), generator=g),
                     torch.randint(0, 8192, (b, s + 1 - 64), generator=g)), dim=1).cuda()
    tokens, labels = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    mask, loss_mask, pos = get_masks_and_position_ids(tokens)
    return (tokens, labels, loss_mask, mask, pos)


def run_step(model, opt, batch, fused):
    from cogview_b200 import pretrain
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    loss, *_ = pretrain.train_step(batch, model, opt, check_skipped=False, fused_loss=fused)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, float(loss)


def part_step(reps):
    model, opt = build_4b(False)
    batch = make_batch(2, 1)
    for fused in (False, True):
        run_step(model, opt, batch, fused)
    res = {False: [], True: []}
    peak = {}
    for _ in range(reps):
        for fused in (False, True):
            torch.cuda.reset_peak_memory_stats()
            ms, loss = run_step(model, opt, batch, fused)
            res[fused].append(ms)
            peak[fused] = torch.cuda.max_memory_allocated()
    for fused in (False, True):
        emit(part="step", route="new" if fused else "old", seqs=2, tokens=2 * 1088,
             ms=round(statistics.median(res[fused]), 1), all_ms=[round(x, 1) for x in res[fused]],
             peak_allocated_gb=round(peak[fused] / 1e9, 2))
    del model, opt, batch
    gc.collect()
    torch.cuda.empty_cache()


def part_fit(max_seqs, reps):
    model, opt = build_4b(True)

    def fits(b, fused):
        """Step times of reps + 1 steps at b sequences (the first one dropped), or None when one runs out of memory."""
        try:
            batch = make_batch(b, 2)
            return [run_step(model, opt, batch, fused)[0] for _ in range(reps + 1)][1:]
        except torch.OutOfMemoryError:
            return None
        finally:
            batch = None
            for p in model.parameters():
                p.grad = None
            gc.collect()
            torch.cuda.empty_cache()

    for fused in (False, True):
        lo, hi, best = 0, None, None
        b = 2
        while b <= max_seqs:
            times = fits(b, fused)
            if times is not None:
                lo, best = b, times
                b *= 2
            else:
                hi = b
                break
        if hi is not None:
            while hi - lo > 1:
                mid = (lo + hi) // 2
                times = fits(mid, fused)
                if times is not None:
                    lo, best = mid, times
                else:
                    hi = mid
        rate = round(lo * 1088 / (statistics.median(best) / 1e3), 1) if lo > 0 else None
        emit(part="fit", route="new" if fused else "old", max_seqs=lo, capped=hi is None, tokens_per_s=rate,
             step_ms=[round(x, 1) for x in best] if best else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="stage,step,fit")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-seqs", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vocab_xent_time.py needs a GPU")
    emit(card=card())
    parts = args.parts.split(",")
    if "stage" in parts:
        part_stage(args.reps)
    if "step" in parts:
        part_step(args.reps)
    if "fit" in parts:
        part_fit(args.max_seqs, max(2, args.reps // 2))


if __name__ == "__main__":
    main()
