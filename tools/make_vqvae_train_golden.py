"""Writes tests/golden/vqvae_train.npz: one training step of the unmodified reference VQVAE (vqvae.api.new_model()
in train() mode, seeded weights of recipes.vqvae_state_dict(seed=0), two seeded 64 x 64 images).

    COGVIEW_REFERENCE=<reference checkout> python tools/make_vqvae_train_golden.py

Recorded: recon, diff and the codes; the gradients of mse(recon, img) + 0.25 diff for all sixteen parameter tensors
(full for the small ones, a fixed strided sample plus the sum and abs-max for the 4 x 4 kernels); the three
quantiser buffers after the step (cluster_size in full, embed and embed_avg at the codes the step used plus a strided
sample).  The CPU restatement tests/vqvae_train_oracle.py is checked against the reference before anything is
written."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import recipes, ref_harness  # noqa: E402
import vqvae_train_oracle as T  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "vqvae_train.npz")
BIG = 4096            # tensors with more elements are stored as strided samples


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref = ref_harness.load()
    sd = recipes.vqvae_state_dict(seed=0)
    img = recipes.images(2, size=64, seed=11)
    model = ref["vq_api"].new_model()
    model.load_state_dict(sd)
    model.train()
    recon, diff = model(img)
    loss = F.mse_loss(recon, img) + T.COMMITMENT * diff.squeeze(0)
    loss.backward()
    with torch.no_grad():
        _, _, codes = T.O.vq_quantize(sd, model.enc_b(img))     # codes of the pre-update codebook, as the step used
    grads = {k: p.grad for k, p in model.named_parameters()}
    bufs = {k: b.detach() for k, b in model.named_buffers()}

    o = T.train_step(sd, img)
    assert torch.equal(o["codes"], codes.view(2, -1)), "oracle codes differ from the reference"
    for name, a, b in [("recon", o["recon"], recon.detach()), ("diff", o["diff"], diff.detach().squeeze(0))] + \
            [(k, o["grads"][k], grads[k]) for k in T.PARAMS] + [(k, o["buffers"][k], bufs[k]) for k in T.BUFFERS]:
        err = (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)
        print("  %-26s rel err %.2e" % (name, err))
        assert err < 1e-6, name

    used = torch.unique(codes.view(-1))
    out = dict(img_seed=np.int64(11), recon=recon.detach().numpy(), diff=np.float32(diff.item()),
               loss=np.float32(loss.item()), codes=codes.view(2, -1).numpy(), used=used.numpy(),
               cluster_size=bufs['quantize_t.cluster_size'].numpy())
    for k in T.PARAMS:
        g = grads[k]
        if g.numel() > BIG:
            out["g/" + k] = T.sample(g).numpy()
            out["gsum/" + k] = np.float64(g.double().sum().item())
            out["gmax/" + k] = np.float32(g.abs().max().item())
        else:
            out["g/" + k] = g.numpy()
    for k in ('quantize_t.embed', 'quantize_t.embed_avg'):
        out["used/" + k] = bufs[k][:, used].numpy()
        out["sample/" + k] = T.sample(bufs[k]).numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "(%d bytes)" % os.path.getsize(OUT))


if __name__ == "__main__":
    main()
