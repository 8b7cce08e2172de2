"""Step time and peak memory of 4B training with the replicated and the sharded (ZeRO stage 1) optimizer.

    python -m torch.distributed.run --nproc_per_node N tools/zero_train_time.py [--reps 5] [--warmup 2]

At the 4B shape (seeded random weights, dropout 0, fused vocabulary loss, no activation recompute), each rank on its
own 1088-token sequences, pretrain.train_step with:
  ddp_fused_b2  : the model in torch DDP (bucket views, 200 MB buckets, as bench.py) + FusedAdamW, 2 sequences per GPU
                  (at N = 1 without the DDP wrapper);
  zero1_b2      : ShardedFusedAdamW (no DDP), 2 sequences per GPU;
  zero1_b4      : ShardedFusedAdamW, 4 sequences per GPU - the reference's train_micro_batch_size_per_gpu.
Per configuration and rank: median step time (host clock around synchronised steps), median time of optimizer.step()
alone (CUDA events; for ZeRO it holds the reduce-scatter, the all-reduce of the norm and the all-gather, which run
after the backward, where DDP overlaps its all-reduce with the backward), torch.cuda.max_memory_allocated, and
whether the configuration ran out of memory.  With N > 1, 8 SMs are kept out of the GEMM grid for NCCL as in
bench.py.  The card's name, power limit and maximum SM clock are read in the same run.  One JSON line per
configuration and rank.  Needs a GPU per rank.
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

SEQ = recipes.COGVIEW_4B["max_sequence_length"] - 1
RESERVED_SMS = 8


def card(dev):
    r = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
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
                              max_sequence_length=cfg["max_sequence_length"], max_memory_length=0,
                              checkpoint_activations=False)
    finally:
        torch.set_default_dtype(old)
    return model.train()


def make_batch(b, seed):
    from cogview_b200.generation.sampling import get_masks_and_position_ids
    g = torch.Generator().manual_seed(seed)
    tok = torch.cat((torch.randint(8192, 58192, (b, 64), generator=g),
                     torch.randint(0, 8192, (b, SEQ + 1 - 64), generator=g)), dim=1).cuda()
    tokens, labels = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    mask, loss_mask, pos = get_masks_and_position_ids(tokens)
    return (tokens, labels, loss_mask, mask, pos)


def run_config(name, world, rank, reps, warmup):
    from cogview_b200 import pretrain
    from cogview_b200.model import PyTorchDistributedDataParallel, gpt2_get_params_for_weight_decay_optimization
    from cogview_b200.optim import FusedAdamW, ShardedFusedAdamW
    b = 4 if name.endswith("b4") else 2
    res = dict(config=name, rank=rank, world=world, seqs_per_gpu=b, tokens_per_gpu=b * SEQ, oom=False)
    model = net = opt = batch = None
    gc.collect()                       # the previous configuration, which an out-of-memory traceback may still hold
    torch.cuda.empty_cache()
    try:
        torch.cuda.reset_peak_memory_stats()
        model = build_4b()
        groups = gpt2_get_params_for_weight_decay_optimization(model)
        kw = dict(lr=1e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_grad_norm=1.0)
        if name.startswith("ddp"):
            opt = FusedAdamW(groups, **kw)
            net = model if world == 1 else PyTorchDistributedDataParallel(
                model, device_ids=[torch.cuda.current_device()], gradient_as_bucket_view=True, bucket_cap_mb=200)
        else:
            opt = ShardedFusedAdamW(groups, **kw)
            net = model
        events = []
        inner = opt.step

        def timed_step():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            inner()
            e1.record()
            events.append((e0, e1))

        opt.step = timed_step
        batch = make_batch(b, 100 + rank)
        times = []
        for i in range(warmup + reps):
            if world > 1:
                torch.distributed.barrier()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pretrain.train_step(batch, net, opt, check_skipped=False, fused_loss=True)
            torch.cuda.synchronize()
            if i >= warmup:
                times.append((time.perf_counter() - t0) * 1e3)
        opt.step = inner
        opt_ms = [e0.elapsed_time(e1) for e0, e1 in events[warmup:]]
        res.update(step_ms=round(statistics.median(times), 1), all_step_ms=[round(x, 1) for x in times],
                   optimizer_step_ms=round(statistics.median(opt_ms), 2),
                   tokens_per_s=round(b * SEQ * world / (statistics.median(times) / 1e3), 1))
    except torch.OutOfMemoryError:
        res["oom"] = True
    res["max_memory_allocated_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", default="ddp_fused_b2,zero1_b2,zero1_b4")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("zero_train_time.py needs a GPU")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(dev)
    if world > 1:
        os.environ.setdefault("NCCL_MAX_CTAS", str(RESERVED_SMS))
        torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", dev))
        from cogview_b200 import _lib
        _lib.lib().cv_set_reserved_sms(RESERVED_SMS)
    print(json.dumps(dict(rank=rank, world=world, card=card(dev))), flush=True)
    for name in args.configs.split(","):
        print(json.dumps(run_config(name, world, rank, args.reps, args.warmup)), flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
