"""The CPU restatement of the Gumbel-softmax quantiser steps (tests/vqvae_gumbel_oracle.py) against the steps of the
unmodified reference recorded in tests/golden/vqvae_gumbel.npz (tools/make_vqvae_gumbel_golden.py), plus the
argument checks of cogview_b200's Quantize that need no GPU."""
import os

import numpy as np
import pytest
import torch

from oracle import recipes
import vqvae_gumbel_oracle as G


def _rel(a, b):
    b = torch.as_tensor(b)
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "vqvae_gumbel.npz"))


CASES = ["soft", "soft_kl", "hard", "hard_kl", "eval_soft"]


def _draws(g, name):
    img = recipes.images(2, size=32, seed=int(g["img_seed"]))
    rows = img.shape[0] * (img.shape[2] // 8) * (img.shape[3] // 8)
    return img, G.exponential_draws(int(g[name + "/noise_seed"]), (rows, 8192))


@pytest.mark.parametrize("name", CASES)
def test_injected_noise_regenerates_exactly(golden, name):
    _, draws = _draws(golden, name)
    assert np.array_equal(G.sample(draws).numpy(), golden[name + "/draws_sample"])
    assert draws.double().sum().item() == float(golden[name + "/draws_sum"])
    assert torch.isfinite(G.gumbels_from_exponential(draws)).all()


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(golden, name):
    g = {k[len(name) + 1:]: golden[k] for k in golden.files if k.startswith(name + "/")}
    assert list(golden["cases"]) == CASES
    img, draws = _draws(golden, name)
    train, hard, use_kl, tau = bool(g["train"]), bool(g["hard"]), bool(g["kl"]), float(g["tau"])
    o = G.train_step(G.state_dict(seed=0), img, G.gumbels_from_exponential(draws), tau, hard, use_kl, training=train)
    assert np.array_equal(o["codes"].numpy(), g["codes"])
    out = o["recon"] if train else o["quant"].permute(0, 3, 1, 2)
    assert _rel(out, g["out"]) < 1e-5
    assert abs(o["diff"].item() - float(g["diff"])) <= 1e-5 * max(abs(float(g["diff"])), 1e-30)
    if not use_kl:
        assert float(g["diff"]) == 0.0
    if not train:
        return
    assert abs(o["loss"].item() - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    stride = int(golden["grad_stride"])
    for k, none in zip(G.PARAMS, g["grad_none"]):
        grad = o["grads"][k]
        assert (grad is None) == bool(none), k
        if grad is None:
            continue
        if "gsum/" + k in g:
            scale = float(g["gmax/" + k])
            assert (G.sample(grad, stride) - torch.as_tensor(g["g/" + k])).abs().max().item() < 1e-5 * scale, k
            assert abs(grad.double().sum().item() - float(g["gsum/" + k])) < 1e-5 * scale * grad.numel() ** 0.5, k
            assert abs(grad.abs().max().item() - scale) < 1e-5 * scale, k
        else:
            assert _rel(grad, g["g/" + k]) < 1e-5, k
    if hard:
        # the reference quirk kept: without the KL the encoder gets no gradient at all
        assert all(o["grads"][k] is None for k in G.PARAMS if k.startswith("enc_b")) == (not use_kl)
        used = torch.as_tensor(g["used"])
        assert _rel(o["buffers"]["quantize_t.cluster_size"], g["cluster_size"]) < 1e-6
        for k in ("quantize_t.embed", "quantize_t.embed_avg"):
            assert _rel(o["buffers"][k][:, used], g["used/" + k]) < 1e-6, k
            assert _rel(G.sample(o["buffers"][k]), g["sample/" + k]) < 1e-6, k
    else:
        sd = G.state_dict(seed=0)
        for k in G.BUFFERS:
            assert torch.equal(o["buffers"][k], sd[k]), k


@pytest.mark.parametrize("tau", [0.0, -1.0])
def test_nonpositive_temperature_is_refused(tau):
    from cogview_b200 import vqvae
    model = vqvae.new_model()
    z = torch.zeros(1, 2, 2, 256)
    for train in (True, False):
        model.train(train)
        with pytest.raises(ValueError, match="temperature"):
            model.quantize_t.forward_(z, continuous_relax=True, temperature=tau)
        with pytest.raises(ValueError, match="temperature"):
            model(torch.zeros(1, 3, 16, 16), continuous_relax=True, temperature=tau, hard=True)
