"""CPU fp32 restatement of one VQ-VAE training step of the reference (vqvae/vqvae_zc.py in train() mode, the hard
nearest-code path of the configuration vqvae.api.new_model() builds), built on the inference restatement in
oracle/cogview_oracle.py.  Used by tests/test_vqvae_train_cpu.py (against the reference's golden step) and
tests/test_vqvae_train_gpu.py (against the CUDA step)."""
import torch
import torch.nn.functional as F

from oracle import cogview_oracle as O

BUFFERS = ('quantize_t.embed', 'quantize_t.cluster_size', 'quantize_t.embed_avg')
PARAMS = ('enc_b.blocks.0.weight', 'enc_b.blocks.0.bias', 'enc_b.blocks.2.weight', 'enc_b.blocks.2.bias',
          'enc_b.blocks.4.weight', 'enc_b.blocks.4.bias', 'enc_b.blocks.6.weight', 'enc_b.blocks.6.bias',
          'dec.blocks.0.weight', 'dec.blocks.0.bias', 'dec.blocks.2.weight', 'dec.blocks.2.bias',
          'dec.blocks.4.weight', 'dec.blocks.4.bias', 'dec.blocks.6.weight', 'dec.blocks.6.bias')
COMMITMENT = 0.25          # loss = mse(recon, img) + 0.25 diff, the VQ-VAE objective the golden step uses


def ema_update(embed, cluster_size, embed_avg, ind, flatten, decay=0.99, eps=1e-5):
    """vqvae_zc.py:67-83 on copies of the three buffers; returns the updated (embed, cluster_size, embed_avg)."""
    n_embed = embed.shape[1]
    onehot = F.one_hot(ind.view(-1), n_embed).type(flatten.dtype)
    embed_onehot_sum = onehot.sum(0)                                       # :68
    embed_sum = flatten.transpose(0, 1) @ onehot                           # :69
    cluster_size = cluster_size.clone().mul_(decay).add_(embed_onehot_sum, alpha=1 - decay)   # :74-76
    embed_avg = embed_avg.clone().mul_(decay).add_(embed_sum, alpha=1 - decay)                # :77
    n = cluster_size.sum()                                                 # :78
    cs = (cluster_size + eps) / (n + n_embed * eps) * n                    # :79-81
    return embed_avg / cs.unsqueeze(0), cluster_size, embed_avg           # :82-83


def train_step(sd, img, codes=None):
    """One step: forward in train() mode, the EMA update and the autograd gradients of
    mse(recon, img) + 0.25 diff.  Returns dict(recon, diff, loss, codes, grads {name: tensor}, buffers {name: tensor}).
    `codes` ([B, h w]) replaces the nearest-code choice, to follow another implementation's codes where near-tied
    distances flip them."""
    p = {k: sd[k].detach().float().clone().requires_grad_(True) for k in PARAMS}
    embed = sd['quantize_t.embed'].float()
    z = O.vq_encoder(p, img)                                               # :117-164, NHWC
    flatten = z.reshape(-1, embed.shape[0])
    _, ind = (-O.vq_distances(flatten, embed)).max(1)                      # :41-51
    if codes is not None:
        ind = codes.reshape(-1).to(ind.device)
    quant = F.embedding(ind, embed.t()).view(z.shape)                      # :53, pre-update codebook
    new_embed, new_cs, new_avg = ema_update(embed, sd['quantize_t.cluster_size'].float(),
                                            sd['quantize_t.embed_avg'].float(), ind, flatten.detach())
    diff = (quant.detach() - z).pow(2).mean()                              # :84
    quantize = z + (quant - z).detach()                                    # :85
    recon = O.vq_decoder(p, quantize.permute(0, 3, 1, 2))                  # :243-247
    loss = F.mse_loss(recon, img) + COMMITMENT * diff
    loss.backward()
    return dict(recon=recon.detach(), diff=diff.detach(), loss=loss.detach(), codes=ind.view(img.shape[0], -1),
                grads={k: p[k].grad for k in PARAMS},
                buffers={'quantize_t.embed': new_embed, 'quantize_t.cluster_size': new_cs,
                         'quantize_t.embed_avg': new_avg})


def sample(t, stride=257):
    """The fixed strided sample of a large tensor stored in the golden fixture."""
    return t.reshape(-1)[::stride]
