"""LayerNorm kernels at the 4B layer shape (4352 x 2560): time and achieved HBM bandwidth.

    python tools/ln_time.py            (COGVIEW_B200_LN_REG=0 selects the shared-memory staged forward kernel)
The inputs (2 x 45 MB) are rotated over 4 copies so that successive launches do not hit in the 50 MB L2."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from cogview_b200 import ops  # noqa: E402


def timeit(fn, n=20):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


def main():
    rows, cols, R = 4352, 2560, 4
    g = torch.Generator(device="cuda").manual_seed(0)
    xf = [torch.randn((rows, cols), generator=g, device="cuda") for _ in range(R)]
    xb = [t.to(torch.bfloat16) for t in xf]
    gamma = torch.ones(cols, dtype=torch.bfloat16, device="cuda")
    beta = torch.zeros(cols, dtype=torch.bfloat16, device="cuda")
    am = torch.full((1,), 5.0, device="cuda")
    amo = torch.zeros(1, device="cuda")
    n = rows * cols
    cases = [
        ("fwd fp32 -> bf16 (LN1 / LN2 / final)", lambda i: ops.layernorm_absmax_fwd(xf[i % R], am, gamma, beta, 1e-5, save_stats=True), n * (4 + 2)),
        ("fwd bf16 + fp32 residual -> fp32 (LN3 / LN4)", lambda i: ops.layernorm_absmax_fwd(
            xb[i % R], am, gamma, beta, 1e-5, residual=xf[(i + 1) % R], out_dtype=torch.float32, absmax_out=amo, save_stats=True), n * (2 + 4 + 4)),
    ]
    _, mean, rstd = ops.layernorm_absmax_fwd(xf[0], am, gamma, beta, 1e-5, save_stats=True)
    cases += [
        ("bwd x fp32, dy bf16 -> dx fp32 (+dres) (LN1 / LN2)", lambda i: ops.layernorm_absmax_bwd(
            xf[i % R], xb[(i + 1) % R], mean, rstd, gamma, dres=xf[(i + 2) % R], dx_dtype=torch.float32), n * (4 + 2 + 4 + 4)),
        ("bwd x bf16, dy fp32 -> dx bf16 (+dxsum) (LN3 / LN4)", lambda i: ops.layernorm_absmax_bwd(
            xb[i % R], xf[(i + 1) % R], mean, rstd, gamma, dx_dtype=torch.bfloat16, want_dxsum=True), n * (2 + 4 + 2)),
    ]
    for name, fn, nbytes in cases:
        us = timeit(fn)
        print("%-55s %7.1f us  %6.0f GB/s (%.0f MB algorithmic)" % (name, us, nbytes / us / 1e3, nbytes / 1e6))


if __name__ == "__main__":
    main()
