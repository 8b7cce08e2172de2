"""Time post-selection (scoring candidate images by their caption's likelihood) at the 4B shape, old route and new.

    python tools/post_selection_time.py [--num 64] [--text 20] [--reps 3]

Seeded random weights at the 4B shape (max_memory_length 1089, mems_mode 'kv'), `num` post-selection rows of one
caption of `text` tokens ([BASE] [BOI1] 1024 codes [EOI1] [ROI1] caption), max_inference_batch_size = num.
  * new : generate.post_selection(..., score=inverse_prompt_scores): GPT2Model.token_logprobs, no logits, no K|V cache;
  * old : generate.post_selection with its default inverse_prompt_score: the full forward (fp32 logits of every
          position, a K|V cache prefilled for the batch), -inf mask, softmax, log.  It is tried at batch `num`, and
          where it runs out of memory at halved batch sizes until one runs.
Per route: time per call (median of --reps calls after one warm-up call, host clock around synchronised calls),
torch.cuda.max_memory_allocated during the calls (and above the weights), and for the old route whether batch `num`
runs and the largest batch that does; the largest |difference| of the two routes' scores.  Then cv_vocab_logprob on
its own at M = num x text rows (CUDA events over 20 launches): TFLOP/s of its 2 M K (V - 8192) operations and the
GB/s of one read of the window's rows of W.  The card's name and power limit are read in the same run.  One JSON line
per measurement.  Needs a GPU.
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


def drop_caches(model):
    tr = model.transformer
    tr.__dict__.pop("_kv_pool", None)
    tr._kv = None
    gc.collect()
    torch.cuda.empty_cache()


def run(model, args, queries, score, reps):
    """(median seconds per call, peak bytes, scores) or None when the route runs out of memory"""
    from cogview_b200 import generate
    drop_caches(model)
    torch.cuda.reset_peak_memory_stats()
    try:
        out = generate.post_selection(model, args, queries, score=score)          # warm-up
        times = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = generate.post_selection(model, args, queries, score=score)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
    except torch.cuda.OutOfMemoryError:
        drop_caches(model)
        return None
    peak = torch.cuda.max_memory_allocated()
    out = out.float().cpu()
    drop_caches(model)
    return statistics.median(times), peak, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num", type=int, default=64)
    ap.add_argument("--text", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("post_selection_time.py needs a GPU")
    from cogview_b200 import generate, ops
    from cogview_b200.generation import sampling
    print(json.dumps(dict(card=card())), flush=True)
    model, cfg = build_model()
    tok = sampling.get_tokenizer()
    torch.cuda.synchronize()
    weights = torch.cuda.memory_allocated()

    class Args:
        is_sparse = 0
        img_tokenizer_num_tokens = 8192
        max_inference_batch_size = a.num

    g = torch.Generator().manual_seed(1)
    text = (8192 + torch.randint(0, 50000, (a.text,), generator=g)).tolist()
    queries = torch.tensor([generate.build_query(generate.QUERY_TEMPLATES['post-selection'],
                                                 [torch.randint(0, 8192, (1024,), generator=g).tolist(), text], tok)
                            for _ in range(a.num)], dtype=torch.long, device="cuda")
    base = dict(num=a.num, text=a.text, seq=queries.shape[1], weights_gb=round(weights / 1e9, 2))

    new = run(model, Args, queries, sampling.inverse_prompt_scores, a.reps)
    print(json.dumps(dict(base, route="new", batch=a.num, ms_per_call=round(new[0] * 1e3, 1),
                          peak_gb=round(new[1] / 1e9, 2), peak_above_weights_gb=round((new[1] - weights) / 1e9, 2))),
          flush=True)

    batch, old = a.num, None
    while batch >= 1:
        Args.max_inference_batch_size = batch
        old = run(model, Args, queries, sampling.inverse_prompt_score, a.reps)
        print(json.dumps(dict(base, route="old", batch=batch, runs=old is not None)), flush=True)
        if old is not None:
            break
        batch //= 2
    if old is not None:
        print(json.dumps(dict(base, route="old", batch=batch, runs_at_num=batch == a.num,
                              ms_per_call=round(old[0] * 1e3, 1), peak_gb=round(old[1] / 1e9, 2),
                              peak_above_weights_gb=round((old[1] - weights) / 1e9, 2),
                              max_abs_score_diff=round((old[2] - new[2]).abs().max().item(), 4),
                              score_scale=round(new[2].abs().max().item(), 2))), flush=True)

    # the kernel alone
    M, K, V = a.num * a.text, cfg["hidden_size"], cfg["vocab_size"]
    w = model.word_embeddings.weight.detach()
    h = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    t = torch.randint(8192, V, (M,), device="cuda")
    for _ in range(3):
        ops.vocab_logprob(h, w, t, 8192, V)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 20
    e0.record()
    for _ in range(n):
        ops.vocab_logprob(h, w, t, 8192, V)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / n
    flop = 2.0 * M * K * (V - 8192)
    w_bytes = (V - 8192) * K * 2
    print(json.dumps(dict(kernel="cv_vocab_logprob", M=M, K=K, window=V - 8192, us=round(us, 1),
                          tflops=round(flop / us / 1e6, 1), w_read_gbps=round(w_bytes / us / 1e3, 1))), flush=True)


if __name__ == "__main__":
    main()
