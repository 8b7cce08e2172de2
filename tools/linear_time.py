"""The four decode linears of a 4B layer (M = 4) back to back, CUDA-graph replayed like the decode step (PDL between
them), L2 flushed by the 157 MB of weights themselves: us per layer-set and achieved HBM bandwidth.

    python tools/linear_time.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from cogview_b200 import ops  # noqa: E402


def main():
    h, M, L = 2560, int(os.environ.get("M", "4")), 8
    g = torch.Generator(device="cuda").manual_seed(0)
    shapes = [("qkv", 3 * h, h), ("dense", h, h), ("fc1", 4 * h, h), ("fc2", h, 4 * h)]
    W = [[(torch.randn((N, K), generator=g, device="cuda") * 0.02).to(torch.bfloat16) for _, N, K in shapes] for _ in range(L)]
    xs = {K: torch.randn((M, K), generator=g, device="cuda").to(torch.bfloat16) for K in (h, 4 * h)}
    outs = {n: torch.empty((M, N), dtype=torch.bfloat16, device="cuda") for n, N, K in shapes}

    def run(which=None):
        for l in range(L):
            for i, (n, N, K) in enumerate(shapes):
                if which is None or which == n:
                    ops.linear_small_m(xs[K], W[l][i], out=outs[n])
    nbytes = sum(N * K * 2 for _, N, K in shapes)
    for which in (None, "qkv", "dense", "fc1", "fc2"):
        run(which); run(which)
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            run(which)
        gr.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            gr.replay()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / 10 / L
        b = nbytes if which is None else [N * K * 2 for n, N, K in shapes if n == which][0]
        print("%-6s %7.2f us per %s  %6.0f GB/s" % (which or "layer", us, "layer (4 linears)" if which is None else "launch", b / us / 1e3))


if __name__ == "__main__":
    main()
