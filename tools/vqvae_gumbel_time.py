"""Times VQ-VAE training with the Gumbel-softmax quantiser on the GPU: a full step (forward in train() mode,
backward, Adam) at 256 x 256 in the soft and hard relaxations, next to the nearest-code step in the same process, with
each step's peak memory; then cv_gumbel_noise, cv_vq_gumbel_fwd and cv_vq_gumbel_bwd alone with CUDA events at the
shapes of that step, with GB/s from the bytes each must move.  Prints the card, its power limit and SM clock first.

    python tools/vqvae_gumbel_time.py [--batch 32] [--size 256] [--steps 5] [--reps 20]
"""
import argparse
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cogview_b200 import ops, recipes, vqvae  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def event_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    B, S = args.batch, args.size
    print("card (name, power limit, SM clock, max SM clock):", card())

    sd = recipes.vqvae_state_dict(seed=0)
    img = recipes.images(B, size=S, seed=1).cuda()
    modes = [("nearest code", dict()),
             ("gumbel soft, KL", dict(continuous_relax=True, temperature=1.0, hard=False, KL=True)),
             ("gumbel soft", dict(continuous_relax=True, temperature=1.0, hard=False, KL=False)),
             ("gumbel hard, KL", dict(continuous_relax=True, temperature=1.0, hard=True, KL=True)),
             ("gumbel hard", dict(continuous_relax=True, temperature=1.0, hard=True, KL=False))]
    for name, kw in modes + modes[:1]:          # the nearest-code step again at the end: the drift of the card
        model = vqvae.new_model()
        model.load_state_dict(sd)
        model = model.cuda().train()
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)

        def step():
            opt.zero_grad(set_to_none=True)
            recon, diff = model(img, **kw)
            (F.mse_loss(recon, img) + 0.25 * diff.squeeze(0)).backward()
            opt.step()

        step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ms = event_ms(step, args.steps, warmup=1)
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        print("full training step, %-16s %d images at %d x %d: %8.2f ms, %6.1f images/s, peak memory %.2f GiB"
              % (name + ":", B, S, S, ms, B * 1000.0 / ms, peak))
        del model, opt

    rows, K = min(16384, B * (S // 8) ** 2), 8192       # one score chunk (Quantize.score_chunk_rows)
    g = torch.Generator(device="cuda").manual_seed(0)
    s = torch.randn(rows, K, generator=g, device="cuda") * 2.0
    e2 = torch.rand(K, generator=g, device="cuda") * 4.0
    dy = torch.randn(rows, K, generator=g, device="cuda")
    n = rows * K
    cases = [("cv_gumbel_noise", lambda: ops.gumbel_noise(7, 0, rows, K), 4 * n),
             ("cv_vq_gumbel_fwd y bf16", lambda: ops.vq_gumbel_fwd(s, e2, 7, 0, 1.0), 4 * n + 2 * n),
             ("cv_vq_gumbel_fwd y bf16 + KL", lambda: ops.vq_gumbel_fwd(s, e2, 7, 0, 1.0, want_kl=True), 6 * n),
             ("cv_vq_gumbel_fwd index only", lambda: ops.vq_gumbel_fwd(s, e2, 7, 0, 1.0, y_dtype=None), 4 * n),
             ("cv_vq_gumbel_fwd index + KL", lambda: ops.vq_gumbel_fwd(s, e2, 7, 0, 1.0, y_dtype=None,
                                                                        want_kl=True), 4 * n),
             ("cv_vq_gumbel_bwd y", lambda: ops.vq_gumbel_bwd(s, e2, 7, 0, 1.0, dy), 4 * n + 4 * n + 2 * n),
             ("cv_vq_gumbel_bwd y + KL", lambda: ops.vq_gumbel_bwd(s, e2, 7, 0, 1.0, dy, 1e-4), 10 * n),
             ("cv_vq_gumbel_bwd KL only", lambda: ops.vq_gumbel_bwd(s, e2, 7, 0, 1.0, None, 1e-4), 4 * n + 2 * n)]
    for name, fn, nbytes in cases:
        t = event_ms(fn, args.reps)
        print("%-30s %d x %d: %8.3f ms  %6.0f GB/s (each input read once, each output written once)"
              % (name, rows, K, t, nbytes / t / 1e6))


if __name__ == "__main__":
    main()
