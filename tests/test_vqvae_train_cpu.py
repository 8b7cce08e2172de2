"""The CPU restatement of one VQ-VAE training step (tests/vqvae_train_oracle.py) against the step of the unmodified
reference recorded in tests/golden/vqvae_train.npz (tools/make_vqvae_train_golden.py): codes exact, gradients within
1e-5 relative, quantiser buffers after the EMA update within 1e-6 relative."""
import os

import numpy as np
import torch

from oracle import recipes
import vqvae_train_oracle as T


def _rel(a, b):
    b = torch.as_tensor(b)
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def test_oracle_training_step_matches_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "vqvae_train.npz"))
    sd = recipes.vqvae_state_dict(seed=0)
    img = recipes.images(2, size=64, seed=int(g["img_seed"]))
    o = T.train_step(sd, img)
    assert np.array_equal(o["codes"].numpy(), g["codes"])
    assert _rel(o["recon"], g["recon"]) < 1e-5
    assert abs(o["diff"].item() - float(g["diff"])) <= 1e-5 * abs(float(g["diff"]))
    assert abs(o["loss"].item() - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    for k in T.PARAMS:
        grad = o["grads"][k]
        if "gsum/" + k in g:
            scale = float(g["gmax/" + k])
            assert (T.sample(grad) - torch.as_tensor(g["g/" + k])).abs().max().item() < 1e-5 * scale, k
            assert abs(grad.double().sum().item() - float(g["gsum/" + k])) < 1e-5 * scale * grad.numel() ** 0.5, k
            assert abs(grad.abs().max().item() - scale) < 1e-5 * scale, k
        else:
            assert _rel(grad, g["g/" + k]) < 1e-5, k
    used = torch.as_tensor(g["used"])
    assert _rel(o["buffers"]["quantize_t.cluster_size"], g["cluster_size"]) < 1e-6
    for k in ("quantize_t.embed", "quantize_t.embed_avg"):
        assert _rel(o["buffers"][k][:, used], g["used/" + k]) < 1e-6, k
        assert _rel(T.sample(o["buffers"][k]), g["sample/" + k]) < 1e-6, k


def test_ema_update_leaves_unused_codes_decayed_only():
    torch.manual_seed(0)
    dim, n = 8, 16
    embed, cs, avg = torch.randn(dim, n), torch.rand(n), torch.randn(dim, n)
    ind = torch.tensor([3, 3, 5])
    flat = torch.randn(3, dim)
    new_embed, new_cs, new_avg = T.ema_update(embed, cs, avg, ind, flat)
    unused = [i for i in range(n) if i not in (3, 5)]
    assert torch.allclose(new_avg[:, unused], 0.99 * avg[:, unused])
    assert torch.allclose(new_cs[3], 0.99 * cs[3] + 0.02)
    assert torch.allclose(new_avg[:, 3], 0.99 * avg[:, 3] + 0.01 * (flat[0] + flat[1]))
