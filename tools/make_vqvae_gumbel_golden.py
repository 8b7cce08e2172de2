"""Writes tests/golden/vqvae_gumbel.npz: steps of the unmodified reference VQVAE with its Gumbel-softmax quantiser
(vqvae.api.new_model(), continuous_relax=True) on the state tests/vqvae_gumbel_oracle.state_dict(seed=0) and two
seeded 32 x 32 images (32 code rows).

    COGVIEW_REFERENCE=<reference checkout> python tools/make_vqvae_gumbel_golden.py

Cases: train() mode soft and hard, each with KL False and True, and one eval-mode soft `encode`.  The reference draws
its noise with torch.Tensor.exponential_ (vqvae_zc.py:332); this tool replaces that method, for the duration of each
case, by one that writes known Exp(1) draws (vqvae_gumbel_oracle.exponential_draws, from numpy's generator, which the
CPU test regenerates).  Recorded per case: recon (or the eval quantize), diff, loss and codes; the gradients of
mse(recon, img) + 0.25 diff (full for small tensors, a strided sample plus the sum and abs-max for large ones, and
which ones are None); the three quantiser buffers in hard mode; a sample and the sum of the injected draws.  The CPU
restatement is checked against the reference (1e-6 relative) before anything is written."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import recipes, ref_harness  # noqa: E402
import vqvae_gumbel_oracle as G  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "vqvae_gumbel.npz")
BIG = 4096            # tensors with more elements are stored as strided samples
STRIDE = 1031         # the sample stride of large gradients (keeps the fixture near 0.5 MB)
IMG_SEED = 11
# (name, hard, KL, train, temperature, noise seed)
CASES = [("soft", False, False, True, 0.5, 101), ("soft_kl", False, True, True, 0.5, 102),
         ("hard", True, False, True, 0.5, 103), ("hard_kl", True, True, True, 0.5, 104),
         ("eval_soft", False, True, False, 1.0, 105)]


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _inject(draws):
    orig = torch.Tensor.exponential_
    calls = []

    def exponential_(self, *args, **kwargs):
        assert tuple(self.shape) == tuple(draws.shape), (self.shape, draws.shape)
        calls.append(1)
        return self.copy_(draws)
    return orig, calls, exponential_


def run_case(ref, sd, img, name, hard, use_kl, train, tau, seed):
    rows = img.shape[0] * (img.shape[2] // 8) * (img.shape[3] // 8)
    draws = G.exponential_draws(seed, (rows, sd['quantize_t.embed'].shape[1]))
    model = ref["vq_api"].new_model()
    model.load_state_dict(sd)
    orig, calls, fake = _inject(draws)
    torch.Tensor.exponential_ = fake
    try:
        if train:
            model.train()
            recon, diff = model(img, continuous_relax=True, temperature=tau, hard=hard, KL=use_kl)
            loss = F.mse_loss(recon, img) + G.COMMITMENT * diff.squeeze(0)
            loss.backward()
            with torch.no_grad():      # the codes: the noise is known, so they follow from the pre-update state
                z = G.O.vq_encoder(sd, img).reshape(rows, -1)
                y = ((-G.O.vq_distances(z, sd['quantize_t.embed']) + G.gumbels_from_exponential(draws)) / tau)
                codes = y.softmax(-1).max(-1)[1]
        else:
            model.eval()
            with torch.no_grad():
                recon, diff, codes = model.encode(img, True, tau, hard, use_kl)
            loss = diff.squeeze(0)
    finally:
        torch.Tensor.exponential_ = orig
    assert len(calls) == 1, "expected one exponential_ draw per step"
    grads = {k: p.grad for k, p in model.named_parameters()}
    bufs = {k: b.detach() for k, b in model.named_buffers()}

    o = G.train_step(sd, img, G.gumbels_from_exponential(draws), tau, hard, use_kl, training=train)
    assert torch.equal(o["codes"].view(-1), codes.reshape(-1)), name + ": oracle codes differ from the reference"
    got_out = o["recon"] if train else o["quant"].permute(0, 3, 1, 2)
    checks = [("out", got_out, recon.detach()), ("diff", o["diff"], diff.detach().squeeze(0))]
    if train:
        checks += [(k, o["grads"][k], grads[k]) for k in G.PARAMS if grads[k] is not None]
        for k in G.PARAMS:
            assert (o["grads"][k] is None) == (grads[k] is None), (name, k)
    checks += [(k, o["buffers"][k], bufs[k]) for k in G.BUFFERS]
    for what, a, b in checks:
        err = _rel(a, b)
        print("  %-10s %-26s rel err %.2e" % (name, what, err))
        assert err < 1e-6, (name, what)
    with torch.no_grad():
        z = G.O.vq_encoder(sd, img).reshape(rows, -1)
        ent, top = G.entropy(-G.O.vq_distances(z, sd['quantize_t.embed']), G.gumbels_from_exponential(draws), tau)
        ent0, _ = G.entropy(-G.O.vq_distances(z, sd['quantize_t.embed']), torch.zeros_like(draws), 1.0)
    print("  %-10s mean row entropy: noised %.3f, noiseless %.3f (uniform %.3f)" % (name, ent, ent0, top))

    out = {"noise_seed": np.int64(seed), "tau": np.float32(tau), "hard": np.bool_(hard), "kl": np.bool_(use_kl),
           "train": np.bool_(train), "out": recon.detach().numpy(), "diff": np.float32(diff.item()),
           "loss": np.float32(loss.item()), "codes": codes.reshape(img.shape[0], -1).numpy(),
           "draws_sample": G.sample(draws).numpy(), "draws_sum": np.float64(draws.double().sum().item())}
    if train:
        out["grad_none"] = np.array([grads[k] is None for k in G.PARAMS])
        for k in G.PARAMS:
            g = grads[k]
            if g is None:
                continue
            if g.numel() > BIG:
                out["g/" + k] = G.sample(g, STRIDE).numpy()
                out["gsum/" + k] = np.float64(g.double().sum().item())
                out["gmax/" + k] = np.float32(g.abs().max().item())
            else:
                out["g/" + k] = g.numpy()
    if hard and train:
        out["cluster_size"] = bufs['quantize_t.cluster_size'].numpy()
        used = torch.unique(codes.reshape(-1))
        out["used"] = used.numpy()
        for k in ('quantize_t.embed', 'quantize_t.embed_avg'):
            out["used/" + k] = bufs[k][:, used].numpy()
            out["sample/" + k] = G.sample(bufs[k]).numpy()
    return {name + "/" + k: v for k, v in out.items()}


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref = ref_harness.load()
    sd = G.state_dict(seed=0)
    img = recipes.images(2, size=32, seed=IMG_SEED)
    out = {"img_seed": np.int64(IMG_SEED), "grad_stride": np.int64(STRIDE), "cases": np.array([c[0] for c in CASES])}
    for case in CASES:
        out.update(run_case(ref, sd, img, *case))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "(%d bytes)" % os.path.getsize(OUT))


if __name__ == "__main__":
    main()
