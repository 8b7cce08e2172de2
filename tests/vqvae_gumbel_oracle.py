"""CPU fp32 restatement of one VQ-VAE step with the reference's Gumbel-softmax quantiser (vqvae/vqvae_zc.py,
Quantize.forward_ with continuous_relax=True: soft :55-60, hard :61-65 with the EMA update :67-83, the KL :87-92,
gumbel_softmax :284-346; VQVAE.encode's zero placeholder :255-258), with the Gumbel noise as an input.  Used by
tests/test_vqvae_gumbel_cpu.py (against the reference's golden steps, tools/make_vqvae_gumbel_golden.py) and
tests/test_vqvae_gumbel_gpu.py (against the CUDA step, on the kernels' own noise)."""
import math

import torch
import torch.nn.functional as F

from oracle import cogview_oracle as O
from oracle import recipes
import vqvae_train_oracle as T

PARAMS, BUFFERS, COMMITMENT = T.PARAMS, T.BUFFERS, T.COMMITMENT
Z_SCALE = 20.0      # scales the encoder's output so that the softmax over the codes is neither uniform nor one-hot


def state_dict(seed=0):
    """recipes.vqvae_state_dict with the encoder's last 1x1 conv scaled by Z_SCALE (with recipes' weights the logits
    -dist of a row differ by ~0.1 and the softmax is uniform to 4 digits) and every code already used once
    (cluster_size 1), the state of a codebook in training rather than a fresh one.  The codebook keeps its scale,
    so the decoder sees inputs of the size the nearest-code training tests use."""
    sd = recipes.vqvae_state_dict(seed=seed)
    for k in ('enc_b.blocks.6.weight', 'enc_b.blocks.6.bias'):
        sd[k] = sd[k] * Z_SCALE
    sd['quantize_t.cluster_size'] = torch.ones_like(sd['quantize_t.cluster_size'])
    return sd


def exponential_draws(seed, shape):
    """The Exp(1) draws the golden tool injects for torch.Tensor.exponential_: -log1p(-u), u ~ numpy's PCG64."""
    import numpy as np
    u = np.random.default_rng(seed).random(size=shape)
    return torch.from_numpy(-np.log1p(-u)).float()


def gumbels_from_exponential(e):
    """vqvae_zc.py:332: g = -log(Exp(1) draw), in fp32."""
    return -e.log()


def gumbel_softmax(logits, gumbels, tau, hard):
    """vqvae_zc.py:333-346 with the noise given: (ret, index)."""
    y = ((logits + gumbels) / tau).softmax(-1)
    index = y.max(-1, keepdim=True)[1]
    if hard:
        y_hard = torch.zeros_like(logits).scatter_(-1, index, 1.0)
        return y_hard - y.detach() + y, index
    return y, index


def kl(logits, n_embed):
    """vqvae_zc.py:89-90."""
    qy = logits.softmax(-1)
    return torch.sum(qy * torch.log(qy * n_embed + 1e-20), dim=-1).mean()


def ema_update(embed, cluster_size, embed_avg, onehot, flatten, decay=0.99, eps=1e-5):
    """vqvae_zc.py:67-83 with the (straight-through) one-hot matrix given; returns (embed, cluster_size, embed_avg)."""
    n_embed = embed.shape[1]
    cluster_size = cluster_size.clone().mul_(decay).add_(onehot.sum(0), alpha=1 - decay)
    embed_avg = embed_avg.clone().mul_(decay).add_(flatten.transpose(0, 1) @ onehot, alpha=1 - decay)
    n = cluster_size.sum()
    cs = (cluster_size + eps) / (n + n_embed * eps) * n
    return embed_avg / cs.unsqueeze(0), cluster_size, embed_avg


def train_step(sd, img, gumbels, tau, hard, use_kl, codes=None, training=True):
    """One forward (train() mode unless training=False) of VQVAE(img, continuous_relax=True, tau, hard, KL=use_kl)
    and the autograd gradients of mse(recon, img) + 0.25 diff.  gumbels: [rows, n_embed] fp32 noise.  `codes`
    replaces the arg-max choice (to follow another implementation's codes where near-ties flip them).
    Returns dict(recon, diff, loss, codes, quant, grads {name: tensor or None}, buffers {name: tensor})."""
    p = {k: sd[k].detach().float().clone().requires_grad_(True) for k in PARAMS}
    # the buffer the reference's autograd reads: its backward of `flatten @ self.embed` (:45) multiplies by the
    # storage of self.embed at backward time, and the hard mode's EMA update writes that storage through .data
    # (:83), which autograd does not see.  So in hard mode the KL gradient goes through the updated codebook.
    embed = sd['quantize_t.embed'].float().clone()
    n_embed = embed.shape[1]
    z = O.vq_encoder(p, img)
    flatten = z.reshape(-1, embed.shape[0])
    logits = -O.vq_distances(flatten, embed)                                 # :43-47
    ret, index = gumbel_softmax(logits, gumbels.to(logits.device), tau, hard)
    if codes is not None:
        index = codes.reshape(-1, 1).to(index.device)
        if hard:
            ret = torch.zeros_like(logits).scatter_(-1, index, 1.0) - ret.detach() + ret.detach()
    ind = index.view(-1)
    if hard:
        quantize = F.embedding(ind, embed.t().clone()).view(z.shape)        # :65, the pre-update codebook
    else:
        quantize = ret.view(*z.shape[:-1], n_embed) @ embed.transpose(0, 1)  # :59-60
    bufs = {k: sd[k].float().clone() for k in BUFFERS}
    if training and hard:
        new_embed, new_cs, new_avg = ema_update(embed, bufs['quantize_t.cluster_size'],
                                                bufs['quantize_t.embed_avg'], ret.detach(), flatten.detach())
        embed.data.copy_(new_embed)
        bufs = {'quantize_t.embed': new_embed, 'quantize_t.cluster_size': new_cs, 'quantize_t.embed_avg': new_avg}
    diff = kl(logits, n_embed)
    if not use_kl:
        diff = torch.zeros_like(diff)                                        # VQVAE.encode :258
    quantize = quantize.to(memory_format=torch.channels_last)                # :92 (only the memory format)
    recon = O.vq_decoder(p, quantize.permute(0, 3, 1, 2))
    loss = F.mse_loss(recon, img) + COMMITMENT * diff
    if training:
        loss.backward()
    return dict(recon=recon.detach(), diff=diff.detach(), loss=loss.detach(), codes=ind.view(img.shape[0], -1),
                quant=quantize.detach(), grads={k: p[k].grad for k in PARAMS}, buffers=bufs)


def entropy(logits, gumbels, tau):
    """Mean row entropy (nats) of the noised, tempered softmax; log(n_embed) is the uniform value."""
    y = ((logits + gumbels) / tau).softmax(-1)
    return -(y * y.clamp_min(1e-38).log()).sum(-1).mean().item(), math.log(logits.shape[-1])


def sample(t, stride=257):
    return T.sample(t, stride)
