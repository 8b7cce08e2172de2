"""VQ-VAE image tokenizer — mirror of the reference's vqvae/vqvae_zc.py for the configuration the reference ships
(`vqvae.api.new_model()`: channel=512, n_res_block=0, embed_dim=256, n_embed=8192, stride=6, simple=True): same
class names, constructor arguments, parameter/buffer names (state_dict keys `enc_b.blocks.{0,2,4,6}`,
`quantize_t.{embed,cluster_size,embed_avg}`, `dec.blocks.{0,2,4,6}`) and method signatures, on the inference
paths `encode` (img -> codes) and `decode_code` (codes -> img).  Training of the VQ-VAE itself (EMA codebook
updates, gumbel relaxation, vqvae_zc.py:55-83, :284-346) is outside the accelerated path and raises.

Device layout: NHWC bf16 activations; the three stride-2 4x4 convolutions and the three transposed convolutions run
as im2col-free wgmma implicit GEMMs (cv_conv2d_k4s2 / cv_conv_transpose2d_k4s2), the Cin=3 first conv as
im2col + GEMM, the 1x1 convs as GEMMs, the quantiser as a 3-term bf16-split tensor-core GEMM + arg-min kernel."""
import torch
from torch import nn

from .. import ops


def _pack_conv(w):        # Conv2d weight [Cout, Cin, 4, 4] -> [16, Cout, Cin]
    return w.detach().permute(2, 3, 0, 1).reshape(16, w.shape[0], w.shape[1]).to(torch.bfloat16).contiguous()


def _pack_convT(w):       # ConvTranspose2d weight [Cin, Cout, 4, 4] -> [16, Cout, Cin]
    return w.detach().permute(2, 3, 1, 0).reshape(16, w.shape[1], w.shape[0]).to(torch.bfloat16).contiguous()


class _PackCache:
    """Re-packed weights, rebuilt when a parameter is modified in place or replaced."""

    def __init__(self):
        self.store = {}

    def get(self, key, tensors, fn):
        sig = tuple((t.data_ptr(), t._version, t.device, t.dtype) for t in tensors)
        hit = self.store.get(key)
        if hit is None or hit[0] != sig:
            hit = (sig, fn())
            self.store[key] = hit
        return hit[1]


class Quantize(nn.Module):
    """vqvae_zc.py:26-96."""

    def __init__(self, dim, n_embed, decay=0.99, eps=1e-5):
        super().__init__()
        self.dim = dim
        self.n_embed = n_embed
        self.decay = decay
        self.eps = eps
        embed = torch.randn(dim, n_embed)
        torch.nn.init.xavier_uniform_(embed, gain=torch.nn.init.calculate_gain('tanh'))
        self.register_buffer("embed", embed)
        self.register_buffer("cluster_size", torch.zeros(n_embed))
        self.register_buffer("embed_avg", embed.clone())
        self._cache = _PackCache()
        self.score_chunk_rows = 16384          # rows of the fp32 score matrix kept alive at once (16 images)

    def _tables(self):
        def build():
            e = self.embed.detach().float()                       # [dim, n_embed]
            et = e.t().contiguous()                               # codebook rows [n_embed, dim]
            hi = et.to(torch.bfloat16)
            lo = (et - hi.float()).to(torch.bfloat16)
            packed = torch.cat((hi, lo, hi), dim=1).contiguous()  # pairs with split3(z) = [hi | hi | lo]
            e2 = e.pow(2).sum(0).contiguous()
            return et, packed, e2
        return self._cache.get("tables", [self.embed], build)

    def forward_(self, input, continuous_relax=False, temperature=1., hard=False):
        if continuous_relax or self.training:
            raise NotImplementedError('only the hard nearest-code inference path is accelerated (eval mode, '
                                      'continuous_relax=False)')
        flatten = input.reshape(-1, self.dim).float().contiguous()
        et, packed, e2 = self._tables()
        idx_parts = []
        for r0 in range(0, flatten.shape[0], self.score_chunk_rows):
            zc = flatten[r0:r0 + self.score_chunk_rows]
            scores = ops.gemm(ops.vq_split3(zc), packed, out_dtype=torch.float32)      # z.E, 16 mantissa bits/operand
            idx_parts.append(ops.vq_argmin(scores, e2, zc, et))
        embed_ind = torch.cat(idx_parts).view(*input.shape[:-1])
        _, quant = ops.vq_lookup(embed_ind, et, want_bf16=False, want_f32=True)
        quantize = quant.view(*input.shape)
        diff = (quantize - input.float()).pow(2).mean()
        return quantize, diff, embed_ind

    def embed_code(self, embed_id):
        et, _, _ = self._tables()
        _, quant = ops.vq_lookup(embed_id, et, want_bf16=False, want_f32=True)
        return quant.view(*embed_id.shape, self.dim)


class Encoder(nn.Module):
    """vqvae_zc.py:117-164 (stride 6, simple): conv k4s2 x3 (+ReLU), ReLU, conv 1x1; output NHWC."""

    def __init__(self, in_channel, channel, n_res_block, n_res_channel, stride, embed_dim, n_embed, simple):
        super().__init__()
        if not (stride == 6 and simple and n_res_block == 0 and in_channel == 3):
            raise NotImplementedError('only the shipped tokenizer configuration (stride=6, simple, no res blocks)')
        self.blocks = nn.Sequential(
            nn.Conv2d(in_channel, channel, 4, stride=2, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(channel, channel, 4, stride=2, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(channel, channel, 4, stride=2, padding=1),
            nn.ReLU(inplace=True), nn.Conv2d(channel, embed_dim, 1))
        self._cache = _PackCache()

    def _packed(self):
        b = self.blocks

        def build():
            w0 = b[0].weight.detach().permute(0, 2, 3, 1).reshape(b[0].weight.shape[0], 48)
            w0p = torch.zeros((w0.shape[0], 64), dtype=torch.bfloat16, device=w0.device)
            w0p[:, :48] = w0.to(torch.bfloat16)
            bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
            return dict(w0=w0p, b0=bf(b[0].bias), w2=_pack_conv(b[2].weight), b2=bf(b[2].bias),
                        w4=_pack_conv(b[4].weight), b4=bf(b[4].bias),
                        w6=bf(b[6].weight.reshape(b[6].weight.shape[0], -1)), b6=bf(b[6].bias))
        return self._cache.get("enc", [b[0].weight, b[0].bias, b[2].weight, b[2].bias, b[4].weight, b[4].bias,
                                       b[6].weight, b[6].bias], build)

    def forward(self, input):
        """input: [B, 3, H, W] (normalised image) -> [B, H/8, W/8, embed_dim] fp32 (NHWC, as the reference returns)."""
        P = self._packed()
        B, _, H, W = input.shape
        ch = P['w0'].shape[0]
        x = ops.gemm(ops.im2col_k4s2_c3(input.float().contiguous()), P['w0'], bias=P['b0'], act=ops.ACT_RELU)
        x = x.view(B, H // 2, W // 2, ch)
        x = ops.conv2d_k4s2(x, P['w2'], P['b2'], relu=True)
        x = ops.conv2d_k4s2(x, P['w4'], P['b4'], relu=True)       # the trailing ReLU of the block list
        z = ops.gemm(x.view(-1, ch), P['w6'], bias=P['b6'], out_dtype=torch.float32)
        return z.view(B, H // 8, W // 8, -1)


class Decoder(nn.Module):
    """vqvae_zc.py:167-214 (stride 4, simple): convT k4s2 x3 (+ReLU), conv 1x1 to 3 channels."""

    def __init__(self, in_channel, out_channel, channel, n_res_block, n_res_channel, stride, simple):
        super().__init__()
        if not (stride == 4 and simple and n_res_block == 0 and out_channel == 3):
            raise NotImplementedError('only the shipped tokenizer configuration (stride=4, simple, no res blocks)')
        self.blocks = nn.Sequential(
            nn.ConvTranspose2d(in_channel, channel, 4, stride=2, padding=1), nn.ReLU(inplace=True),
            nn.ConvTranspose2d(channel, channel, 4, stride=2, padding=1), nn.ReLU(inplace=True),
            nn.ConvTranspose2d(channel, channel, 4, stride=2, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(channel, out_channel, 1))
        self._cache = _PackCache()
        # images per pass at 256 x 256 output, where the last activation is 67 MB / image in bf16; larger outputs
        # take proportionally fewer images per pass (4 at 512 x 512)
        self.batch_chunk = 16

    def _packed(self):
        b = self.blocks

        def build():
            bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
            return dict(w0=_pack_convT(b[0].weight), b0=bf(b[0].bias), w2=_pack_convT(b[2].weight), b2=bf(b[2].bias),
                        w4=_pack_convT(b[4].weight), b4=bf(b[4].bias),
                        w6=b[6].weight.detach().reshape(3, -1).float().contiguous(), b6=b[6].bias.detach().float())
        return self._cache.get("dec", [b[0].weight, b[0].bias, b[2].weight, b[2].bias, b[4].weight, b[4].bias,
                                       b[6].weight, b[6].bias], build)

    def forward_nhwc(self, quant_nhwc, scale=None, shift=None):
        """quant_nhwc: [B, h, w, C] bf16 -> [B, 3, 8h, 8w] fp32 (optionally de-normalised: out * scale + shift)."""
        P = self._packed()
        dev = quant_nhwc.device
        one = torch.ones(3, device=dev) if scale is None else scale
        zero = torch.zeros(3, device=dev) if shift is None else shift
        h, w = quant_nhwc.shape[1], quant_nhwc.shape[2]
        chunk = max(1, min(self.batch_chunk, self.batch_chunk * 256 * 256 // (8 * h * 8 * w)))
        outs = []
        for b0 in range(0, quant_nhwc.shape[0], chunk):
            x = quant_nhwc[b0:b0 + chunk].contiguous()
            x = ops.conv_transpose2d_k4s2(x, P['w0'], P['b0'], relu=True)
            x = ops.conv_transpose2d_k4s2(x, P['w2'], P['b2'], relu=True)
            x = ops.conv_transpose2d_k4s2(x, P['w4'], P['b4'], relu=True)
            outs.append(ops.conv1x1_out3(x, P['w6'], P['b6'], one, zero))
        return outs[0] if len(outs) == 1 else torch.cat(outs)

    def forward(self, input):
        """input: [B, C, h, w] (NCHW, as the reference) -> [B, 3, 8h, 8w]."""
        return self.forward_nhwc(input.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous())


class VQVAE(nn.Module):
    """vqvae_zc.py:217-269."""

    def __init__(self, in_channel=3, channel=128, n_res_block=2, n_res_channel=32, embed_dim=64, n_embed=1024,
                 stride=4, simple=True, decay=0.99):
        super().__init__()
        if channel == 2048:
            n_res_block = 0
        self.enc_b = Encoder(in_channel, channel, n_res_block, n_res_channel, stride, embed_dim, n_embed, simple)
        self.quantize_t = Quantize(embed_dim, n_embed)
        self.dec = Decoder(in_channel=embed_dim, out_channel=in_channel, channel=channel, n_res_block=n_res_block,
                           n_res_channel=n_res_channel, stride=stride - 2, simple=simple)

    def forward(self, input, continuous_relax=False, temperature=1., hard=False, KL=False):
        quant_t, diff, _ = self.encode(input, continuous_relax, temperature, hard, KL)
        return self.dec(quant_t), diff

    def encode(self, input, continuous_relax=False, temperature=1., hard=False, KL=False):
        logits = self.enc_b(input)
        quant_t, diff_t, id_t = self.quantize_t.forward_(logits, continuous_relax, temperature, hard)
        return quant_t.permute(0, 3, 1, 2), diff_t.unsqueeze(0), id_t

    def decode(self, code):
        return self.dec(code)

    def decode_code(self, code_t, scale=None, shift=None):
        et, _, _ = self.quantize_t._tables()
        quant, _ = ops.vq_lookup(code_t, et, want_bf16=True, want_f32=False)          # embed_code + NHWC layout
        return self.dec.forward_nhwc(quant.view(*code_t.shape, -1), scale, shift)
