"""VQ-VAE image tokenizer — mirror of the reference's vqvae/vqvae_zc.py for the configuration the reference ships
(`vqvae.api.new_model()`: channel=512, n_res_block=0, embed_dim=256, n_embed=8192, stride=6, simple=True): same
class names, constructor arguments, parameter/buffer names (state_dict keys `enc_b.blocks.{0,2,4,6}`,
`quantize_t.{embed,cluster_size,embed_avg}`, `dec.blocks.{0,2,4,6}`) and method signatures, on the inference
paths `encode` (img -> codes) and `decode_code` (codes -> img), and in train() mode `forward` (img -> recon, diff)
with the EMA codebook update (vqvae_zc.py:67-83) and a backward for every parameter.  The Gumbel-softmax
relaxations (continuous_relax=True: soft :55-60, hard :61-65 with the EMA update, the KL :87-92, gumbel_softmax
:284-346) run in train and eval mode, with `KL` passed through VQVAE.forward / encode.  Their noise is Gumbel(0, 1)
from a counter-based Philox stream under one seed per call drawn from torch's default generator: the same
distribution as the reference's torch.exponential_ draws, not the same numbers.

Device layout: NHWC bf16 activations; the three stride-2 4x4 convolutions and the three transposed convolutions run
as im2col-free wgmma implicit GEMMs (cv_conv2d_k4s2 / cv_conv_transpose2d_k4s2), the Cin=3 first conv as
im2col + GEMM, the 1x1 convs as GEMMs, the quantiser as a 3-term bf16-split tensor-core GEMM + arg-min kernel.
Training: one autograd Function per network half (_EncoderFn, _DecoderFn) saves the bf16 ReLU outputs; data gradients
run on the forward convolution kernels with the adjoint packing (the data gradient of Conv2d(k4, s2, p1) is
ConvTranspose2d(k4, s2, p1) with the same weight, and the reverse) followed by the ReLU mask, weight gradients on
cv_conv_k4s2_wgrad and the GEMM's wgrad operand modes, bias gradients on cv_colsum_bf16.  Relaxed quantiser: the
split3 score GEMM, then cv_vq_gumbel_fwd (noised tempered softmax y, arg-max, KL) and y @ E^T on the GEMM; its
backward (_GumbelFn) recomputes the scores from the saved z and runs dq @ E, cv_vq_gumbel_bwd and da @ E^T."""
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

    def _gumbel_tables(self):
        """bf16 codebook E [dim, n_embed] (the GEMM operand of y @ E^T and da @ E^T) and E^T [n_embed, dim] (dq @ E)."""
        return self._cache.get("gumbel", [self.embed],
                               lambda: (self.embed.detach().to(torch.bfloat16).contiguous(),
                                        self.embed.detach().t().to(torch.bfloat16).contiguous()))

    def forward_(self, input, continuous_relax=False, temperature=1., hard=False, kl=True):
        """vqvae_zc.py:41-93.  `kl` (not in the reference) is False when the caller discards the KL, as VQVAE.encode
        does without KL=True: diff is then the zero placeholder of :258 and the KL is not computed."""
        if continuous_relax:
            return self._forward_relaxed(input, temperature, hard, kl)
        if self.training:
            return self._forward_train(input)
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

    def _nearest(self, flatten):
        et, packed, e2 = self._tables()
        idx_parts = []
        for r0 in range(0, flatten.shape[0], self.score_chunk_rows):
            zc = flatten[r0:r0 + self.score_chunk_rows]
            scores = ops.gemm(ops.vq_split3(zc), packed, out_dtype=torch.float32)
            idx_parts.append(ops.vq_argmin(scores, e2, zc, et))
        return torch.cat(idx_parts), et

    def _forward_train(self, input):
        """vqvae_zc.py:41-54, :67-86 (hard path): the code is chosen and looked up with the codebook as it was before
        this step's EMA update; then cluster_size, embed_avg and embed are updated in place, in the reference's order."""
        flatten = input.detach().reshape(-1, self.dim).float().contiguous()
        embed_ind, et = self._nearest(flatten)
        _, quant = ops.vq_lookup(embed_ind, et, want_bf16=False, want_f32=True)
        quant = quant.view(*input.shape)
        self._ema_update(embed_ind, flatten)
        diff = (quant - input).pow(2).mean()
        quantize = input + (quant - input).detach()        # straight-through estimator
        return quantize, diff, embed_ind.view(*input.shape[:-1])

    def _ema_update(self, embed_ind, flatten):
        """vqvae_zc.py:67-83 from the chosen codes and the fp32 rows they were chosen for."""
        embed_onehot_sum, embed_sum = ops.vq_ema_stats(embed_ind, flatten, self.n_embed)
        with torch.no_grad():
            self.cluster_size.mul_(self.decay).add_(embed_onehot_sum, alpha=1 - self.decay)
            self.embed_avg.mul_(self.decay).add_(embed_sum, alpha=1 - self.decay)
            n = self.cluster_size.sum()
            cluster_size = (self.cluster_size + self.eps) / (n + self.n_embed * self.eps) * n
            self.embed.copy_(self.embed_avg / cluster_size.unsqueeze(0))

    def _forward_relaxed(self, input, temperature, hard, kl):
        """vqvae_zc.py:55-65, :67-83 (hard only, in train() mode), :87-92.  The noise comes from the kernels' counter
        stream under one seed drawn from torch's default generator per call (torch.manual_seed repeats a run)."""
        _check_temperature(temperature)
        seed = int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())
        flatten = input.reshape(-1, self.dim)
        if hard and not kl:        # nothing differentiable leaves: the lookup carries no gradient (:65)
            quant, _, embed_ind = _gumbel_forward(flatten.detach().float().contiguous(), self, seed, float(temperature), True, False)
            diff = torch.zeros((), dtype=torch.float32, device=input.device)
        else:
            quant, diff, embed_ind = _GumbelFn.apply(flatten, self, seed, float(temperature), hard, kl)
        if self.training and hard:
            self._ema_update(embed_ind, flatten.detach().float().contiguous())
        return quant.view(*input.shape), diff, embed_ind.view(*input.shape[:-1])

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

    def _packed_bwd(self):
        b = self.blocks
        # the data gradient of Conv2d(k4, s2, p1) is ConvTranspose2d(k4, s2, p1) with the same weight tensor
        return self._cache.get("enc_bwd", [b[2].weight, b[4].weight],
                               lambda: dict(w2=_pack_convT(b[2].weight), w4=_pack_convT(b[4].weight)))

    def forward(self, input):
        """input: [B, 3, H, W] (normalised image) -> [B, H/8, W/8, embed_dim] fp32 (NHWC, as the reference returns)."""
        if self.training:
            return _EncoderFn.apply(input, self, *[t for m in self.blocks[0::2] for t in (m.weight, m.bias)])
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

    def _packed_bwd(self):
        b = self.blocks
        # the data gradient of ConvTranspose2d(k4, s2, p1) is Conv2d(k4, s2, p1) with the same weight tensor
        return self._cache.get("dec_bwd", [b[0].weight, b[2].weight, b[4].weight],
                               lambda: dict(w0=_pack_conv(b[0].weight), w2=_pack_conv(b[2].weight),
                                            w4=_pack_conv(b[4].weight)))

    def forward(self, input):
        """input: [B, C, h, w] (NCHW, as the reference) -> [B, 3, 8h, 8w]."""
        if self.training:
            return _DecoderFn.apply(input.permute(0, 2, 3, 1), self,
                                    *[t for m in self.blocks[0::2] for t in (m.weight, m.bias)])
        return self.forward_nhwc(input.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous())


def _bias_grad(g2d):
    return ops.colsum(g2d).float()


class _EncoderFn(torch.autograd.Function):
    """Encoder forward (the kernels of Encoder.forward in eval mode, without batch chunking) and its backward for the
    eight parameters.  Saved: the first conv's im2col patches and the three bf16 ReLU outputs."""

    @staticmethod
    def forward(ctx, img, enc, *params):
        P = enc._packed()
        B, _, H, W = img.shape
        ch = P['w0'].shape[0]
        a0 = ops.im2col_k4s2_c3(img.detach().float().contiguous())
        x1 = ops.gemm(a0, P['w0'], bias=P['b0'], act=ops.ACT_RELU).view(B, H // 2, W // 2, ch)
        x2 = ops.conv2d_k4s2(x1, P['w2'], P['b2'], relu=True)
        x3 = ops.conv2d_k4s2(x2, P['w4'], P['b4'], relu=True)
        z = ops.gemm(x3.view(-1, ch), P['w6'], bias=P['b6'], out_dtype=torch.float32)
        ctx.save_for_backward(a0, x1, x2, x3)
        ctx.P, ctx.PT = P, enc._packed_bwd()
        return z.view(B, H // 8, W // 8, -1)

    @staticmethod
    def backward(ctx, dz):
        a0, x1, x2, x3 = ctx.saved_tensors
        P, PT = ctx.P, ctx.PT
        ch = x3.shape[-1]
        dz = dz.to(torch.bfloat16).contiguous().view(-1, dz.shape[-1])               # [pixels, embed_dim]
        dw6 = ops.gemm(dz, x3.view(-1, ch), a_mn_major=True, b_mn_major=True, out_dtype=torch.float32)
        db6 = _bias_grad(dz)
        g3 = ops.relu_mask_(ops.gemm(dz, P['w6'], b_mn_major=True), x3.view(-1, ch)).view(x3.shape)
        dw4 = ops.conv_k4s2_wgrad(g3, x2)
        db4 = _bias_grad(g3.view(-1, ch))
        g2 = ops.relu_mask_(ops.conv_transpose2d_k4s2(g3, PT['w4'], None, relu=False), x2)
        dw2 = ops.conv_k4s2_wgrad(g2, x1)
        db2 = _bias_grad(g2.view(-1, ch))
        g1 = ops.relu_mask_(ops.conv_transpose2d_k4s2(g2, PT['w2'], None, relu=False), x1).view(-1, ch)
        # first conv through its im2col matrix: columns (ky * 4 + kx) * 3 + c of the 64 (48 used)
        dw0 = ops.gemm(g1, a0, a_mn_major=True, b_mn_major=True, out_dtype=torch.float32)[:, :48]
        dw0 = dw0.reshape(ch, 4, 4, 3).permute(0, 3, 1, 2).contiguous()
        db0 = _bias_grad(g1)
        return (None, None, dw0, db0, dw2, db2, dw4, db4, dw6.view(dw6.shape[0], ch, 1, 1), db6)


class _DecoderFn(torch.autograd.Function):
    """Decoder forward (the kernels of Decoder.forward_nhwc, without batch chunking) from NHWC fp32 quant and its
    backward for the eight parameters and for quant.  Saved: the bf16 input and the three bf16 ReLU outputs."""

    @staticmethod
    def forward(ctx, quant_nhwc, dec, *params):
        P = dec._packed()
        dev = quant_nhwc.device
        x0 = quant_nhwc.detach().to(torch.bfloat16).contiguous()
        a1 = ops.conv_transpose2d_k4s2(x0, P['w0'], P['b0'], relu=True)
        a2 = ops.conv_transpose2d_k4s2(a1, P['w2'], P['b2'], relu=True)
        a3 = ops.conv_transpose2d_k4s2(a2, P['w4'], P['b4'], relu=True)
        out = ops.conv1x1_out3(a3, P['w6'], P['b6'], torch.ones(3, device=dev), torch.zeros(3, device=dev))
        ctx.save_for_backward(x0, a1, a2, a3)
        ctx.P, ctx.PT = P, dec._packed_bwd()
        return out

    @staticmethod
    def backward(ctx, dout):
        x0, a1, a2, a3 = ctx.saved_tensors
        P, PT = ctx.P, ctx.PT
        ch = a3.shape[-1]
        g3, dw6, db6 = ops.conv1x1_out3_bwd(dout.float().contiguous(), a3, P['w6'])
        dw4 = ops.conv_k4s2_wgrad(a2, g3)
        db4 = _bias_grad(g3.view(-1, ch))
        g2 = ops.relu_mask_(ops.conv2d_k4s2(g3, PT['w4'], None, relu=False), a2)
        dw2 = ops.conv_k4s2_wgrad(a1, g2)
        db2 = _bias_grad(g2.view(-1, ch))
        g1 = ops.relu_mask_(ops.conv2d_k4s2(g2, PT['w2'], None, relu=False), a1)
        dw0 = ops.conv_k4s2_wgrad(x0, g1)
        db0 = _bias_grad(g1.view(-1, ch))
        dq = None
        if ctx.needs_input_grad[0]:
            dq = ops.conv2d_k4s2(g1, PT['w0'], None, relu=False).float()
        return (dq, None, dw0, db0, dw2, db2, dw4, db4, dw6.view(3, ch, 1, 1), db6)


def _check_temperature(temperature):
    # the reference divides by it unchecked and returns inf or NaN for tau <= 0
    if not temperature > 0:
        raise ValueError('the Gumbel-softmax temperature must be positive, got %r' % (temperature,))


def _gumbel_forward(z, q, seed, tau, hard, kl):
    """The relaxed quantiser on fp32 rows z [rows, dim], score_chunk_rows rows at a time: the split3 score GEMM, then
    cv_vq_gumbel_fwd.  Soft: quant = y @ E^T (bf16 y, bf16 E, fp32 accumulation).  Hard: quant = the code's row of
    the current codebook.  Returns (quant [rows, dim] fp32, the KL mean (or None), idx [rows])."""
    et, packed, e2 = q._tables()
    e_bf, _ = q._gumbel_tables()
    rows = z.shape[0]
    quant = None if hard else torch.empty((rows, q.dim), dtype=torch.float32, device=z.device)
    idx, kls = [], []
    for r0 in range(0, rows, q.score_chunk_rows):
        zc = z[r0:r0 + q.score_chunk_rows]
        scores = ops.gemm(ops.vq_split3(zc), packed, out_dtype=torch.float32)
        y, i, k = ops.vq_gumbel_fwd(scores, e2, seed, r0, tau, y_dtype=None if hard else torch.bfloat16, want_kl=kl)
        del scores
        if not hard:
            ops.gemm(y, e_bf, out_dtype=torch.float32, out=quant[r0:r0 + zc.shape[0]])
        idx.append(i)
        kls.append(k)
    idx = torch.cat(idx)
    if hard:
        _, quant = ops.vq_lookup(idx, et, want_bf16=False, want_f32=True)
    return quant, (torch.cat(kls).mean() if kl else None), idx


class _GumbelFn(torch.autograd.Function):
    """The relaxed quantiser of Quantize.forward_ (vqvae_zc.py:55-65, :89-90) and its backward to z.  Saved: z and
    the seed; the scores, y and qy are recomputed in the backward, score_chunk_rows rows at a time.

    Backward, as the reference's autograd computes it: with a = -dist, dL/da from cv_vq_gumbel_bwd (the y term from
    dy = dq @ E in soft mode, the KL term when the KL is in the loss), then dz = 2 da @ E^T - 2 z rowsum(da).  The
    scores are those of the forward's codebook; the two GEMMs with E read the codebook as it is at backward time,
    because the reference's matmul backward reads the buffer, which its hard-mode EMA update rewrites through .data
    in between (:83)."""

    @staticmethod
    def forward(ctx, z, q, seed, tau, hard, kl):
        zd = z.detach().float().contiguous()
        quant, diff, idx = _gumbel_forward(zd, q, seed, tau, hard, kl)
        if diff is None:
            diff = torch.zeros((), dtype=torch.float32, device=z.device)
            ctx.mark_non_differentiable(diff)
        if hard:
            ctx.mark_non_differentiable(quant)
        ctx.mark_non_differentiable(idx)
        ctx.save_for_backward(zd)
        _, packed, e2 = q._tables()
        ctx.scores_tables = (packed, e2)
        ctx.q, ctx.seed, ctx.tau, ctx.hard, ctx.kl = q, seed, tau, hard, kl
        return quant, diff, idx

    @staticmethod
    def backward(ctx, dq, ddiff, _didx):
        (z,) = ctx.saved_tensors
        q = ctx.q
        rows = z.shape[0]
        want_y = not ctx.hard and dq is not None
        kl_scale = float(ddiff) / rows if (ctx.kl and ddiff is not None) else 0.0
        if not want_y and kl_scale == 0.0:
            return None, None, None, None, None, None
        packed, e2 = ctx.scores_tables
        e_bf, et_bf = q._gumbel_tables()
        dqb = dq.reshape(rows, q.dim).to(torch.bfloat16).contiguous() if want_y else None
        dz = torch.empty_like(z)
        for r0 in range(0, rows, q.score_chunk_rows):
            zc = z[r0:r0 + q.score_chunk_rows]
            r1 = r0 + zc.shape[0]
            scores = ops.gemm(ops.vq_split3(zc), packed, out_dtype=torch.float32)
            dy = ops.gemm(dqb[r0:r1], et_bf, out_dtype=torch.float32) if want_y else None
            da, rowsum = ops.vq_gumbel_bwd(scores, e2, ctx.seed, r0, ctx.tau, dy, kl_scale)
            del scores, dy
            g = ops.gemm(da, e_bf, out_dtype=torch.float32)                   # da @ E^T
            dz[r0:r1] = 2.0 * (g - zc * rowsum.unsqueeze(1))
        return dz, None, None, None, None, None


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
        if not continuous_relax:
            logits = self.enc_b(input)
            quant_t, diff_t, id_t = self.quantize_t.forward_(logits, continuous_relax, temperature, hard)
            return quant_t.permute(0, 3, 1, 2), diff_t.unsqueeze(0), id_t
        _check_temperature(temperature)
        logits = self.enc_b(input)
        # without KL the reference returns zeros_like(diff) (:255-258); the KL is then not computed
        quant_t, diff_t, id_t = self.quantize_t.forward_(logits, True, temperature, hard, kl=KL)
        return quant_t.permute(0, 3, 1, 2), diff_t.unsqueeze(0), id_t

    def decode(self, code):
        return self.dec(code)

    def decode_code(self, code_t, scale=None, shift=None):
        et, _, _ = self.quantize_t._tables()
        quant, _ = ops.vq_lookup(code_t, et, want_bf16=True, want_f32=False)          # embed_code + NHWC layout
        return self.dec.forward_nhwc(quant.view(*code_t.shape, -1), scale, shift)
