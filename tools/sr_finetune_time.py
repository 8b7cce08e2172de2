"""Step time and peak memory of 4B super-resolution finetuning on 2121-token two-image rows.

    python tools/sr_finetune_time.py [--reps 5] [--warmup 2] [--out FILE]

At the 4B shape (seeded random weights, dropout 0, dense attention), rows of 2121 tokens as
data.make_super_resolution_batch writes them for a 64-id text ([ROI1] text [BASE] [BOI1] 1024 codes [EOI1] [ROI2]
[POSi] [BASE] [BOI2] 1024 codes [EOI2]; the codes are seeded stand-ins for the VQ-VAE's) go through
data.make_batch(args=finetune) - positions restarting at [ROI2], clamped to the 1089-entry table - and
pretrain.train_step with the fused vocabulary loss and FusedAdamW, at 1, 2 and 4 rows per step, with activation
recompute (checkpoint_activations) off and on.  Per configuration: median step time (host clock around
synchronised steps), trained tokens per second (2120 per row), torch.cuda.max_memory_allocated, and whether it ran out
of memory.  The card's name, power limit and maximum SM clock are read in the same run.  One JSON line per
configuration (also appended to --out).  Needs a GPU.
"""
import argparse
import gc
import json
import os
import random
import statistics
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from cogview_b200 import recipes  # noqa: E402

MPE, MPE_FT = recipes.COGVIEW_4B["max_sequence_length"], 2121
FT = types.SimpleNamespace(finetune=True, max_position_embeddings=MPE, max_position_embeddings_finetune=MPE_FT)


def card():
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def build_4b():
    from cogview_b200.model import GPT2Model
    cfg = recipes.COGVIEW_4B
    torch.manual_seed(0)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            model = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"],
                              hidden_size=cfg["hidden_size"], num_attention_heads=cfg["num_attention_heads"],
                              embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                              max_sequence_length=MPE, max_memory_length=0, checkpoint_activations=False)
    finally:
        torch.set_default_dtype(old)
    return model.train()


def sr_batch(b, seed):
    from cogview_b200 import data as D
    g = torch.Generator().manual_seed(seed)
    texts = [(8192 + torch.randint(0, 50000, (64,), generator=g)).tolist() for _ in range(b)]
    random.seed(seed)
    rows = D.make_super_resolution_batch(None, texts, torch.zeros(b, 3, 512, 512), sampling_num=1,
                                         encode=lambda x: torch.randint(0, 8192, (x.shape[0], 1024), generator=g))
    assert all(len(r) == MPE_FT for r in rows)
    fn = D.filled_tokenized_process_fn(MPE_FT)
    items = [fn(r.numpy()) for r in rows]
    return D.make_batch({k: np.stack([it[k] for it in items]) for k in ('text', 'loss_mask')}, device="cuda",
                        args=FT)


def run_config(model, opt, b, ckpt, reps, warmup):
    from cogview_b200 import pretrain
    res = dict(rows=b, row_tokens=MPE_FT, checkpoint_activations=ckpt, fused_loss=True, oom=False)
    batch = None
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    try:
        model.transformer.checkpoint_activations = ckpt
        batch = sr_batch(b, 100 + b)
        times = []
        for i in range(warmup + reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loss, skipped, _, _, _ = pretrain.train_step(batch, model, opt, fused_loss=True)
            torch.cuda.synchronize()
            if i >= warmup:
                times.append((time.perf_counter() - t0) * 1e3)
        ms = statistics.median(times)
        res.update(step_ms=round(ms, 1), all_step_ms=[round(x, 1) for x in times],
                   tokens_per_s=round(b * (MPE_FT - 1) / (ms / 1e3), 1), last_loss=round(float(loss), 4),
                   skipped=int(skipped))
    except torch.OutOfMemoryError:
        res["oom"] = True
    batch = None
    model.zero_grad(set_to_none=True)
    res["max_memory_allocated_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rows", default="1,2,4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sr_finetune_time.py needs a GPU")
    from cogview_b200.model import gpt2_get_params_for_weight_decay_optimization
    from cogview_b200.optim import FusedAdamW
    lines = [dict(card=card(), torch=torch.__version__)]
    print(json.dumps(lines[0]), flush=True)
    model = build_4b()
    opt = FusedAdamW(gpt2_get_params_for_weight_decay_optimization(model), lr=1e-5, betas=(0.9, 0.999), eps=1e-8,
                     weight_decay=0.01, max_grad_norm=1.0)
    for ckpt in (False, True):
        for b in [int(x) for x in args.rows.split(",")]:
            lines.append(run_config(model, opt, b, ckpt, args.reps, args.warmup))
            print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
