"""Times VQ-VAE training on the GPU: a full step (forward in train() mode, EMA update, backward, Adam) at 256 x 256,
and each training kernel alone with CUDA events at the shapes of that step.  FLOP/s of the weight gradients and
bytes/s of the memory-bound kernels are computed from the shapes.  Prints the card and its power limit first.

    python tools/vqvae_train_time.py [--batch 32] [--size 256] [--steps 5] [--reps 20]
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
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
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
    print("card:", card())

    model = vqvae.new_model()
    model.load_state_dict(recipes.vqvae_state_dict(seed=0))
    model = model.cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    img = recipes.images(B, size=S, seed=1).cuda()

    def step():
        opt.zero_grad(set_to_none=True)
        recon, diff = model(img)
        (F.mse_loss(recon, img) + 0.25 * diff.squeeze(0)).backward()
        opt.step()

    ms = event_ms(step, args.steps, warmup=2)
    print("full training step, %d images at %d x %d: %.2f ms, %.1f images/s" % (B, S, S, ms, B * 1000.0 / ms))

    g = torch.Generator(device="cuda").manual_seed(0)

    def bf16(*shape):
        return torch.randn(shape, generator=g, device="cuda").relu().to(torch.bfloat16)

    # weight gradients: (layer, small-map channels, big-map channels, small-map side)
    for name, m, n, side in [("enc conv2 512->512", 512, 512, S // 4), ("enc conv4 512->512", 512, 512, S // 8),
                             ("dec convT0 256->512", 256, 512, S // 8), ("dec convT2 512->512", 512, 512, S // 4),
                             ("dec convT4 512->512", 512, 512, S // 2)]:
        s, gg = bf16(B, side, side, m), bf16(B, 2 * side, 2 * side, n)
        t = event_ms(lambda: ops.conv_k4s2_wgrad(s, gg), args.reps)
        flop = 2.0 * 16 * m * n * B * side * side
        print("cv_conv_k4s2_wgrad %-20s small map %4d: %8.3f ms  %6.1f TFLOP/s" % (name, side, t, flop / t / 1e9))
        del s, gg

    x = bf16(B, S, S, 512)
    dr = torch.randn(B, 3, S, S, generator=g, device="cuda")
    w = torch.randn(3, 512, generator=g, device="cuda") * 0.05
    t = event_ms(lambda: ops.conv1x1_out3_bwd(dr, x, w), args.reps)
    nbytes = x.numel() * 2 * 2 + dr.numel() * 4
    print("cv_conv1x1_out3_bwd %d x %d x 512: %.3f ms  %.0f GB/s" % (S, S, t, nbytes / t / 1e6))
    dx = x.clone()
    t = event_ms(lambda: ops.relu_mask_(dx, x), args.reps)
    print("cv_relu_mask_bf16 %d elements: %.3f ms  %.0f GB/s" % (x.numel(), t, 3 * x.numel() * 2 / t / 1e6))
    del x, dx, dr

    rows = B * (S // 8) ** 2
    z = torch.randn(rows, 256, generator=g, device="cuda")
    idx = torch.randint(0, 8192, (rows,), generator=g, device="cuda")
    t = event_ms(lambda: ops.vq_ema_stats(idx, z, 8192), args.reps)
    nbytes = z.numel() * 4 + rows * 8 + 8192 * 257 * 4
    print("cv_vq_ema_stats %d rows: %.3f ms  %.0f GB/s (z, codes and outputs once)" % (rows, t, nbytes / t / 1e6))


if __name__ == "__main__":
    main()
