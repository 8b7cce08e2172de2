"""VQ-VAE training on the GPU (train() mode of cogview_b200.vqvae): the k4 s2 weight-gradient kernel, the adjoint
reuse of the forward convolution kernels for data gradients, the deterministic EMA codebook statistics, a whole
step against the fp32 restatement, and a short Adam run."""
import pytest
import torch
import torch.nn.functional as F

from oracle import cogview_oracle as O
from oracle import recipes
import vqvae_train_oracle as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def fp32_reference():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _bf16(shape, seed, relu=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, generator=g, device="cuda")
    return (x.relu() if relu else x).to(torch.bfloat16)


def _nchw(t):
    return t.float().permute(0, 3, 1, 2).contiguous()


# (layer, kind, small-map channels, big-map channels, small-map size at a 64 x 64 image)
LAYERS = [("enc2", "conv", 512, 512, 16), ("enc4", "conv", 512, 512, 8), ("dec0", "convT", 256, 512, 8),
          ("dec2", "convT", 512, 512, 16), ("dec4", "convT", 512, 512, 32)]
WGRAD_CASES = [(name, kind, m, n, B, s * scale, s * scale)
               for name, kind, m, n, s in LAYERS for scale in (1, 4) for B in (1, 8)]
WGRAD_CASES.append(("rowseg", "convT", 512, 512, 1, 8, 256))        # a map wider than 128


def _torch_wgrad(kind, s, g):
    """fp32 autograd weight gradient; for conv (s, g) = (dY, X), for convT (s, g) = (X, dY)."""
    if kind == "conv":
        w = torch.zeros(s.shape[3], g.shape[3], 4, 4, device="cuda", requires_grad=True)
        y = F.conv2d(_nchw(g), w, stride=2, padding=1)
        (gw,) = torch.autograd.grad(y, w, _nchw(s))
    else:
        w = torch.zeros(s.shape[3], g.shape[3], 4, 4, device="cuda", requires_grad=True)
        y = F.conv_transpose2d(_nchw(s), w, stride=2, padding=1)
        (gw,) = torch.autograd.grad(y, w, _nchw(g))
    return gw


@pytest.mark.parametrize("name,kind,m,n,B,h,w", WGRAD_CASES)
def test_wgrad_kernel(name, kind, m, n, B, h, w):
    from cogview_b200 import ops
    s = _bf16((B, h, w, m), 1, relu=(kind == "convT"))
    g = _bf16((B, 2 * h, 2 * w, n), 2, relu=(kind == "conv"))
    got = ops.conv_k4s2_wgrad(s, g)
    ref = _torch_wgrad(kind, s, g)
    scale = ref.abs().max().item()
    assert (got - ref).abs().max().item() <= 1e-2 * scale
    assert torch.equal(got, ops.conv_k4s2_wgrad(s, g)), "not deterministic"


ADJOINT_CASES = [(name, kind, m, n, s * scale) for name, kind, m, n, s in LAYERS for scale in (1, 4)]


@pytest.mark.parametrize("name,kind,m,n,h", ADJOINT_CASES)
def test_adjoint_data_gradient(name, kind, m, n, h):
    """Data gradients through the forward kernels with swapped packing, then the ReLU mask of the saved activation."""
    from cogview_b200 import ops
    from cogview_b200.vqvae.vqvae_zc import _pack_conv, _pack_convT
    B = 2
    gen = torch.Generator().manual_seed(3)
    if kind == "conv":            # Conv2d(n -> m): x [B, 2h, 2h, n] (a ReLU output), dy [B, h, h, m]
        wt = ((torch.rand(m, n, 4, 4, generator=gen) * 2 - 1) / (16 * n) ** 0.5).cuda()
        x = _bf16((B, 2 * h, 2 * h, n), 4, relu=True)
        dy = _bf16((B, h, h, m), 5)
        dx = ops.relu_mask_(ops.conv_transpose2d_k4s2(dy, _pack_convT(wt), None, relu=False), x)
        xin = _nchw(x).requires_grad_(True)
        (ref,) = torch.autograd.grad(F.conv2d(xin, wt.bfloat16().float(), stride=2, padding=1), xin, _nchw(dy))
    else:                         # ConvTranspose2d(m -> n): x [B, h, h, m] (a ReLU output), dy [B, 2h, 2h, n]
        wt = ((torch.rand(m, n, 4, 4, generator=gen) * 2 - 1) / (16 * m) ** 0.5).cuda()
        x = _bf16((B, h, h, m), 4, relu=True)
        dy = _bf16((B, 2 * h, 2 * h, n), 5)
        dx = ops.relu_mask_(ops.conv2d_k4s2(dy, _pack_conv(wt), None, relu=False), x)
        xin = _nchw(x).requires_grad_(True)
        (ref,) = torch.autograd.grad(F.conv_transpose2d(xin, wt.bfloat16().float(), stride=2, padding=1), xin,
                                     _nchw(dy))
    ref = ref * (_nchw(x) > 0)
    scale = ref.abs().max().item()
    assert (_nchw(dx) - ref).abs().max().item() <= 1e-2 * scale


def test_conv1x1_out3_bwd():
    from cogview_b200 import ops
    x = _bf16((2, 64, 64, 512), 6, relu=True)
    dr = torch.randn(2, 3, 64, 64, device="cuda")
    w = torch.randn(3, 512, device="cuda") * 0.05
    dx, dw, db = ops.conv1x1_out3_bwd(dr, x, w)
    xf = _nchw(x)
    ref_dx = torch.einsum("bchw,ci->bihw", dr, w) * (xf > 0)
    ref_dw = torch.einsum("bchw,bihw->ci", dr.double(), xf.double()).float()
    assert (_nchw(dx) - ref_dx).abs().max().item() <= 1e-2 * ref_dx.abs().max().item()
    assert (dw - ref_dw).abs().max().item() <= 1e-4 * ref_dw.abs().max().item()
    assert torch.allclose(db, dr.double().sum((0, 2, 3)).float(), rtol=1e-4, atol=1e-3)
    dx2, dw2, db2 = ops.conv1x1_out3_bwd(dr, x, w)
    assert torch.equal(dx, dx2) and torch.equal(dw, dw2) and torch.equal(db, db2)


@pytest.mark.parametrize("case", ["random", "one_code"])
def test_ema_stats(case):
    from cogview_b200 import ops
    rows, dim, n_embed = 4096, 256, 8192
    g = torch.Generator(device="cuda").manual_seed(7)
    z = torch.randn(rows, dim, generator=g, device="cuda")
    if case == "random":          # codes 0 .. 2047 only: most codes have no rows
        idx = torch.randint(0, 2048, (rows,), generator=g, device="cuda")
    else:
        idx = torch.full((rows,), 4321, dtype=torch.int64, device="cuda")
    counts, esum = ops.vq_ema_stats(idx, z, n_embed)
    onehot = F.one_hot(idx, n_embed).double()
    ref_counts = onehot.sum(0)
    ref_sum = z.double().t() @ onehot
    assert torch.equal(counts.double(), ref_counts)
    assert (esum.double() - ref_sum).abs().max().item() <= 1e-5 * ref_sum.abs().max().item()
    counts2, esum2 = ops.vq_ema_stats(idx, z, n_embed)
    assert torch.equal(counts, counts2) and torch.equal(esum, esum2)


def _model(sd):
    from cogview_b200 import vqvae
    m = vqvae.new_model()
    m.load_state_dict(sd)
    return m.cuda().train()


@pytest.mark.parametrize("size,batch", [(64, 8), (256, 2)])
def test_whole_step_matches_oracle(size, batch):
    sd = recipes.vqvae_state_dict(seed=0)
    img = recipes.images(batch, size=size, seed=11).cuda()
    model = _model(sd)
    with torch.no_grad():
        z = model.enc_b(img).reshape(-1, 256).clone()             # the z the step's statistics are taken over
        codes, _ = model.quantize_t._nearest(z)                  # with the codebook before the update
    recon, diff = model(img)
    loss = F.mse_loss(recon, img) + T.COMMITMENT * diff.squeeze(0)
    loss.backward()
    # the kernels compute with bf16 copies of the weights: the restatement gets the same rounded weights.  A code
    # that flips between near-tied distances changes a whole row of the straight-through gradient, so the gradients
    # are compared with the restatement following the CUDA run's codes; agreement with its own choice is reported.
    sdr = {k: (v if k in T.BUFFERS else v.bfloat16().float()).cuda() for k, v in sd.items()}
    free = T.train_step(sdr, img)
    agree = (codes.view(batch, -1) == free["codes"]).float().mean().item()
    o = T.train_step(sdr, img, codes=codes)
    print("size %d: loss %.5f vs oracle %.5f, codes agreeing %.4f" % (size, loss.item(), free["loss"].item(), agree))
    assert abs(loss.item() - free["loss"].item()) <= 1e-2 * max(1.0, abs(free["loss"].item()))
    assert agree >= 0.9
    params = dict(model.named_parameters())
    errs = {}
    for k in T.PARAMS:
        ref = o["grads"][k]
        assert params[k].grad.dtype == torch.float32, k
        errs[k] = (params[k].grad - ref).abs().max().item() / ref.abs().max().item()
        print("  %-24s grad err %.2e of scale, %.2e in norm" % (k, errs[k], ((params[k].grad - ref).norm() /
                                                                           ref.norm()).item()))
    assert max(errs.values()) <= 6e-2, errs
    # the EMA update, restated on the CUDA run's own codes and z
    e, cs, avg = T.ema_update(sd['quantize_t.embed'].cuda(), sd['quantize_t.cluster_size'].cuda(),
                              sd['quantize_t.embed_avg'].cuda(), codes, z)
    q = model.quantize_t
    for got, ref in ((q.cluster_size, cs), (q.embed_avg, avg), (q.embed, e)):
        assert (got - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


def test_adam_steps_reduce_loss_and_eval_still_matches():
    sd = recipes.vqvae_state_dict(seed=0)
    # smooth images with a mean offset, which the tokenizer can learn to reconstruct
    img = F.interpolate(recipes.images(4, size=8, seed=12), scale_factor=8, mode="bilinear") + 0.5
    img = img.cuda().contiguous()
    model = _model(sd)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        recon, diff = model(img)
        loss = F.mse_loss(recon, img) + T.COMMITMENT * diff.squeeze(0)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print("losses", ["%.4f" % v for v in losses])
    assert losses[-1] < 0.9 * losses[0], losses
    model.eval()
    from cogview_b200 import vqvae
    sd2 = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    codes = vqvae.img2code(model, img)
    o_codes = O.img2code(sd2, img.cpu())
    agree = (codes.cpu() == o_codes).float().mean().item()
    print("eval codes agreeing with the oracle after 20 steps: %.4f" % agree)
    assert agree >= 0.9
    rec = vqvae.code2img(model, codes.view(4, 8, 8))
    o_rec = O.code2img(sd2, codes.cpu().view(4, 8, 8))
    assert (rec.cpu() - o_rec).abs().max().item() <= 3e-2 * o_rec.abs().max().item()
