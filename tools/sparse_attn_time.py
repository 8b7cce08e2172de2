"""Times cv_attn_sparse_fwd + cv_attn_sparse_bwd at the CogView-sr training shape (b=2, 40 heads, s=4096, w=128, times=6,
768 pivots), without and with attention-probability dropout (p = 0.1), the two alternated in one process.  Prints the
keep-bit buffer size, the card and its power limit."""
import os
import random
import subprocess
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from cogview_b200 import _lib, ops


def timeit(fn, n=20):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / n


def main():
    b, heads, s, w, times, n_piv = 2, 40, 4096, 128, 6, 768
    h = heads * 64
    random.seed(0)
    torch.manual_seed(0)
    qkv = torch.randn((b, s, 3 * h), device="cuda").to(torch.bfloat16)
    d_out = torch.randn((b, s, h), device="cuda").to(torch.bfloat16)
    q, k, v = qkv[..., :h], qkv[..., h:2 * h], qkv[..., 2 * h:]
    piv = torch.stack([torch.tensor(sorted(random.sample(range(s), n_piv))) for _ in range(b)]).cuda()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    words = _lib.lib().cv_attn_sparse_drop_mask_words(b, heads, s, n_piv, w, times)
    print("card: %s" % gpu)
    print("shape b=%d heads=%d s=%d w=%d times=%d n_piv=%d; keep bits %.1f MB (%.2f MB per sequence and head)" % (
        b, heads, s, w, times, n_piv, words * 4 / 2 ** 20, words * 4 / 2 ** 20 / (b * heads)))

    def step(p):
        if p > 0:
            out, lse, mask = ops.attn_sparse_fwd(q, k, v, heads, piv, w, times, want_lse=True, dropout=(p, 1234, 3))
        else:
            (out, lse), mask = ops.attn_sparse_fwd(q, k, v, heads, piv, w, times, want_lse=True), None
        ops.attn_sparse_bwd(q, k, v, out, d_out, lse, heads, piv, w, times, dropout_p=p, drop_mask=mask)

    for p in (0.0, 0.1):
        for _ in range(3):
            step(p)
    res = {0.0: [], 0.1: []}
    for _ in range(10):                 # alternate the two so that clock and neighbour drift hit both alike
        for p in (0.0, 0.1):
            res[p].append(timeit(lambda: step(p)))
    for p, ts in res.items():
        ts.sort()
        print("dropout %.1f: fwd + bwd median %.1f us (min %.1f, max %.1f over %d windows of 20)" % (
            p, ts[len(ts) // 2], ts[0], ts[-1], len(ts)))
    m0, m1 = sorted(res[0.0])[5], sorted(res[0.1])[5]
    print("dropout overhead: %.1f%%" % (100.0 * (m1 / m0 - 1.0)))


if __name__ == "__main__":
    main()
