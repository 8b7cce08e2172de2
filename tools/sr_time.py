"""Times the super-resolution path on one GPU and prints the card and its power limit.

  1. vqvae.code2img per image at 32 x 32 codes (256 x 256 output, 16 images per call) and at 64 x 64 codes
     (512 x 512 output, 4 images per call), with achieved TFLOP/s from the convolution shapes;
  2. the k4 s2 convolutions alone at equal pixel counts on whole-row tiles (tile grid 128 wide) and on row-segment
     tiles (tile grid 256 wide), 512 channels, alternated;
  3. one generate.super_resolution call (nine magnify windows, 4096 codes, one 512 x 512 image) on the 4B shape
     (48 layers, h = 2560, 40 heads, seeded random weights), top-k 200, temperature 1.02 as in the reference's script.

Every shape is warmed up first.  Times are medians over windows of at least a second (device events around the
window); the super-resolution call is longer than that on its own and is timed by a synchronised host clock.

    python tools/sr_time.py [--sr-calls 3] [--skip-sr]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cogview_b200 import generate, ops, recipes, vqvae  # noqa: E402
from cogview_b200.generation import sampling  # noqa: E402


def window_ms(fn, windows=5, min_s=1.0):
    """median ms per call over `windows` windows, each of enough calls to last at least min_s."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    n = max(1, int(min_s * 1e3 / max(a.elapsed_time(b), 1e-3)) + 1)
    res = []
    for _ in range(windows):
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        res.append(a.elapsed_time(b) / n)
    return statistics.median(res), min(res), max(res), n


def decoder_flops(h, w, embed_dim=256, ch=512):
    """code grid h x w -> image 8h x 8w: three k4 s2 transposed convs (4 taps per output pixel) and the 1x1 to RGB."""
    f = 2 * (2 * h * 2 * w) * ch * 4 * embed_dim
    f += 2 * (4 * h * 4 * w) * ch * 4 * ch
    f += 2 * (8 * h * 8 * w) * ch * 4 * ch
    f += 2 * (8 * h * 8 * w) * 3 * ch
    return f


def time_code2img(model):
    print("code2img (decode of code grids, de-normalised fp32 image out):")
    g = torch.Generator().manual_seed(0)
    cases = [(32, 16), (64, 4)]
    inputs = {s: torch.randint(0, 8192, (n, s, s), generator=g).cuda() for s, n in cases}
    with torch.no_grad():
        for s, _ in cases:                                  # warm-up of every shape
            vqvae.code2img(model, inputs[s])
        torch.cuda.synchronize()
        for s, n in cases:
            med, lo, hi, calls = window_ms(lambda: vqvae.code2img(model, inputs[s]))
            per = med / n
            tf = decoder_flops(s, s) / (per * 1e-3) / 1e12
            print("  %dx%d codes -> %dx%d: %.3f ms per image (median; %d images per call, windows of %d calls, "
                  "%.3f .. %.3f ms per call), %.1f TFLOP/s, %.2f ns per output pixel" % (
                      s, s, 8 * s, 8 * s, per, n, calls, lo, hi, tf, per * 1e6 / (64 * s * s)))


def time_conv_kernels():
    print("k4 s2 convolutions, 512 -> 512 channels, equal output pixels (alternated):")
    g = torch.Generator().manual_seed(1)
    w = (torch.randn((16, 512, 512), generator=g) * 0.02).to(torch.bfloat16).cuda()
    bias = torch.randn(512, generator=g).to(torch.bfloat16).cuda()

    def x(b, hh, ww):
        return torch.randn((b, hh, ww, 512), generator=g).to(torch.bfloat16).cuda()
    cases = [
        ("convT whole rows,   input 4 x 128 x 128", ops.conv_transpose2d_k4s2, x(4, 128, 128), 4 * 256 * 256),
        ("convT row segments, input 1 x 256 x 256", ops.conv_transpose2d_k4s2, x(1, 256, 256), 256 * 256 * 4),
        ("conv  whole rows,   input 4 x 256 x 256", ops.conv2d_k4s2, x(4, 256, 256), 4 * 128 * 128),
        ("conv  row segments, input 1 x 512 x 512", ops.conv2d_k4s2, x(1, 512, 512), 256 * 256),
    ]
    for _, fn, xi, _ in cases:
        fn(xi, w, bias, relu=True)
    torch.cuda.synchronize()
    res = {name: [] for name, *_ in cases}
    for _ in range(5):
        for name, fn, xi, _ in cases:
            res[name].append(window_ms(lambda: fn(xi, w, bias, relu=True), windows=1)[0])
    for name, fn, xi, out_px in cases:
        taps = 4 if fn is ops.conv_transpose2d_k4s2 else 16
        med = statistics.median(res[name])
        print("  %s: %.3f ms (median of 5 windows; %.3f .. %.3f), %.1f TFLOP/s" % (
            name, med, min(res[name]), max(res[name]), 2 * out_px * 512 * taps * 512 / (med * 1e-3) / 1e12))


class SRArgs:
    temperature = 1.02
    top_k = 200
    top_p = 0.0
    is_sparse = 0
    img_tokenizer_num_tokens = 8192


def time_super_resolution(vq_model, calls):
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
                              max_sequence_length=cfg["max_sequence_length"], max_memory_length=1345,
                              checkpoint_activations=False)
    finally:
        torch.set_default_dtype(old)
    model.eval()
    tok = sampling.get_tokenizer(SRArgs)
    g = torch.Generator().manual_seed(2)
    text = torch.randint(8192, 58192, (20,), generator=g).tolist()
    src = torch.randint(0, 8192, (1024,), generator=g).tolist()
    seq = torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['super-resolution'], [text, src], tokenizer=tok),
                       dtype=torch.long, device="cuda")
    print("super_resolution, 4B shape (%d layers, h=%d, %d heads, V=%d), %d-token template, top-k %d, T %.2f:" % (
        cfg["num_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["vocab_size"], len(seq), SRArgs.top_k,
        SRArgs.temperature))
    times = []
    for i in range(calls + 1):                             # the first call is the warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        codes, imgs = generate.super_resolution(model, vq_model, SRArgs, seq)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        assert codes.shape == (1, 4096) and imgs.shape == (1, 3, 512, 512)
        print("  call %d%s: %.2f s" % (i, " (warm-up)" if i == 0 else "", dt))
        if i > 0:
            times.append(dt)
    print("  median %.2f s per 512 x 512 image over %d calls (4096 sampled codes: %.2f ms per code)" % (
        statistics.median(times), len(times), statistics.median(times) * 1e3 / 4096))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sr-calls", type=int, default=3)
    ap.add_argument("--skip-sr", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sr_time.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card (name, power limit, max SM clock): %s; torch device: %s" % (card, torch.cuda.get_device_name()))
    vq_model = vqvae.new_model()
    vq_model.load_state_dict(recipes.vqvae_state_dict(seed=0))
    vq_model = vq_model.cuda().eval()
    time_code2img(vq_model)
    time_conv_kernels()
    if not args.skip_sr:
        time_super_resolution(vq_model, args.sr_calls)


if __name__ == "__main__":
    main()
