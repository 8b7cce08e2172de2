"""Super-resolution on the GPU: the VQ-VAE convolutions on maps wider than 128 (row-segment tiles), the decoder at
64 x 64 codes (512 x 512 images), the encoder at 512 x 512 images, and generate.super_resolution end to end through a
small GPT2Model and the real-shaped VQ-VAE.

References are float32 CPU computations on the bf16-rounded inputs and weights the kernels see.  Errors are measured
per output row (one image row of one image, all its columns and channels) against that row's own scale, so a wrong
tile cannot hide behind a large value elsewhere.  Every input is seeded."""
import pytest
import torch
import torch.nn.functional as F

from oracle import cogview_oracle as O
from oracle import recipes

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


def bfr(t):
    return t.to(BF16).float()


def row_err(got, want, rows, floor=0.0):
    """max over `rows` equal slices of max|got - want| / max|want| of the slice.  floor > 0 raises every slice's
    scale to at least that fraction of the whole tensor's scale."""
    got = got.detach().double().cpu().reshape(rows, -1)
    want = want.detach().double().cpu().reshape(rows, -1)
    scale = want.abs().amax(-1).clamp_min(floor * want.abs().max().item()).clamp_min(1e-300)
    return ((got - want).abs().amax(-1) / scale).max().item()


# ----------------------------------------------------------------------------------------------------
# convolution kernels on wide maps vs torch.nn.functional on the CPU
# ----------------------------------------------------------------------------------------------------
# (Cin, Cout, batch, relu, bias): every value of every factor, both BN instantiations (Cout 128 -> BN 128,
# Cout 256 -> BN 256) with and without ReLU and bias
CASES = [(64, 128, 1, True, True), (128, 256, 2, False, False), (64, 256, 2, True, False), (128, 128, 1, False, True)]


def _conv_inputs(seed, B, Cin, Cout, H, W, transposed, bias):
    g = torch.Generator().manual_seed(seed)
    x = bfr(torch.randn((B, Cin, H, W), generator=g))
    wshape = (Cin, Cout, 4, 4) if transposed else (Cout, Cin, 4, 4)
    w = bfr(torch.randn(wshape, generator=g) * 0.05)
    b = bfr(torch.randn(Cout, generator=g)) if bias else None
    return x, w, b


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("H,W", [(512, 512), (256, 1024)])
def test_conv2d_k4s2_wide_output(ops, H, W, case):
    """input H x W -> output H/2 x W/2 with W/2 = 256 or 512: row-segment tiles of 128 output columns."""
    from cogview_b200.vqvae.vqvae_zc import _pack_conv
    Cin, Cout, B, relu, bias = case
    x, w, b = _conv_inputs(H + W + Cin + Cout + B, B, Cin, Cout, H, W, False, bias)
    ref = F.conv2d(x, w, b, stride=2, padding=1)
    if relu:
        ref = ref.relu()
    y = ops.conv2d_k4s2(x.permute(0, 2, 3, 1).to(BF16).contiguous().cuda(), _pack_conv(w).cuda(),
                        None if b is None else b.to(BF16).cuda(), relu=relu)
    torch.cuda.synchronize()
    assert y.shape == (B, H // 2, W // 2, Cout)
    err = row_err(y.float().cpu().permute(0, 3, 1, 2).transpose(1, 2), ref.transpose(1, 2), B * (H // 2))
    print("conv2d %dx%d Cin %d Cout %d B %d relu %d bias %d: row err %.3e" % (H, W, Cin, Cout, B, relu, bias, err))
    assert err < 1e-2


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("H,W", [(256, 256), (256, 512)])
def test_conv_transpose2d_k4s2_wide_input(ops, H, W, case):
    """input H x W with W = 256 or 512 -> output 2H x 2W: each phase tiles its input rows in 128-column segments."""
    from cogview_b200.vqvae.vqvae_zc import _pack_convT
    Cin, Cout, B, relu, bias = case
    x, w, b = _conv_inputs(7 * H + W + Cin + Cout + B, B, Cin, Cout, H, W, True, bias)
    ref = F.conv_transpose2d(x, w, b, stride=2, padding=1)
    if relu:
        ref = ref.relu()
    y = ops.conv_transpose2d_k4s2(x.permute(0, 2, 3, 1).to(BF16).contiguous().cuda(), _pack_convT(w).cuda(),
                                  None if b is None else b.to(BF16).cuda(), relu=relu)
    torch.cuda.synchronize()
    assert y.shape == (B, 2 * H, 2 * W, Cout)
    err = row_err(y.float().cpu().permute(0, 3, 1, 2).transpose(1, 2), ref.transpose(1, 2), B * 2 * H)
    print("convT %dx%d Cin %d Cout %d B %d relu %d bias %d: row err %.3e" % (H, W, Cin, Cout, B, relu, bias, err))
    assert err < 1e-2


@pytest.mark.parametrize("W", [96, 192, 320])
def test_untileable_widths_are_refused(ops, W):
    """Tile grids 96 wide (<= 128, not a power of two), 192 and 320 wide (> 128, not multiples of 128)."""
    from cogview_b200._lib import CogViewB200Error
    x = torch.zeros((1, 8, 2 * W, 64), dtype=BF16, device="cuda")
    w = torch.zeros((16, 128, 64), dtype=BF16, device="cuda")
    with pytest.raises(CogViewB200Error, match=r"output W must be a power of two <= 128 \(with H a power of two and "
                                               r"128 pixels tiling the batch\) or a multiple of 128"):
        ops.conv2d_k4s2(x, w, None, relu=False)
    xt = torch.zeros((1, 4, W, 64), dtype=BF16, device="cuda")
    with pytest.raises(CogViewB200Error, match=r"input W must be a power of two <= 128 \(with H a power of two and "
                                               r"128 pixels tiling the batch\) or a multiple of 128"):
        ops.conv_transpose2d_k4s2(xt, w, None, relu=False)


# ----------------------------------------------------------------------------------------------------
# the VQ-VAE at 512 x 512 (new_model() shapes)
# ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def vq():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import vqvae
    sd = recipes.vqvae_state_dict(seed=0)
    model = vqvae.new_model()
    model.load_state_dict(sd)
    return dict(model=model.cuda().eval(), sd=sd, vqvae=vqvae)


def _sd_bf16(sd, prefixes):
    return {k: (bfr(v) if k.startswith(prefixes) else v) for k, v in sd.items()}


def test_decoder_at_64x64_codes(vq):
    m, sd, vqvae = vq["model"], vq["sd"], vq["vqvae"]
    codes = torch.randint(0, 8192, (1, 64, 64), generator=torch.Generator().manual_seed(21))
    with torch.no_grad():
        rec = vqvae.code2img(m, codes.cuda()).cpu()
        raw = m.decode_code(codes.cuda()).cpu()
    assert rec.shape == raw.shape == (1, 3, 512, 512)
    # the kernels see bf16 codebook rows and bf16 transposed-conv weights; the final 1x1 runs in fp32
    q = bfr(F.embedding(codes, sd["quantize_t.embed"].t()))
    sdb = _sd_bf16(sd, ("dec.blocks.0.", "dec.blocks.2.", "dec.blocks.4."))
    raw_ref = O.vq_decoder(sdb, q.permute(0, 3, 1, 2))
    std = torch.tensor(O.IMG_STD).view(1, 3, 1, 1)
    mean = torch.tensor(O.IMG_MEAN).view(1, 3, 1, 1)
    rec_ref = raw_ref * std + mean
    rel = ((raw - raw_ref).abs().max() / raw_ref.abs().max()).item()
    rel_rows = row_err(raw, raw_ref, 3 * 512, floor=0.1)
    img = ((rec - rec_ref).abs().max() / rec_ref.abs().max()).item()
    img_rows = row_err(rec, rec_ref, 3 * 512)
    print("512x512 decoder: pre-denorm rel err %.3e (per row %.3e), image err %.3e of scale (per row %.3e)" % (
        rel, rel_rows, img, img_rows))
    assert rel < 2e-2 and rel_rows < 2e-2
    assert img < 3e-2 and img_rows < 3e-2


def test_encoder_and_codes_at_512x512(vq):
    """z within 2e-2 of its scale; codes equal wherever the reference's nearest / second-nearest distance gap exceeds
    the bound the bf16 encoder error puts on a distance (2 |dz| |e_i - e_j| <= 4 |dz| max|e|), as in
    tests/test_vqvae_gpu.py at 256 x 256."""
    m, sd, vqvae = vq["model"], vq["sd"], vq["vqvae"]
    img = bfr(recipes.images(1, size=512, seed=9))
    with torch.no_grad():
        z = m.enc_b(img.cuda()).float().cpu()
        codes = vqvae.img2code(m, img.cuda()).cpu().view(-1)
    sdb = _sd_bf16(sd, ("enc_b.",))
    z_ref = O.vq_encoder(sdb, img)
    assert z.shape == z_ref.shape == (1, 64, 64, 256)
    dz = (z - z_ref).abs().max().item()
    zrows = row_err(z, z_ref, 64)
    print("512x512 encoder: |dz| max %.3e (z scale %.3f), per row %.3e" % (dz, z_ref.abs().max().item(), zrows))
    assert dz < 2e-2 * z_ref.abs().max().item() and zrows < 2e-2
    embed = sd["quantize_t.embed"]
    d = O.vq_distances(z_ref.reshape(-1, embed.shape[0]), embed)
    top2 = torch.topk(-d, 2, dim=1)
    ref_codes = top2.indices[:, 0]
    gap = top2.values[:, 0] - top2.values[:, 1]
    emax = embed.abs().sum(0).max().item()
    decisive = gap > 4.0 * dz * emax
    agree = codes == ref_codes
    print("512x512: code agreement %.4f (%d of %d); decisive codes %d, all equal: %s" % (
        agree.float().mean().item(), agree.sum().item(), agree.numel(), decisive.sum().item(),
        bool(agree[decisive].all())))
    assert agree[decisive].all()
    assert agree.float().mean().item() > 0.9


def test_chunked_decode_at_512_matches_single_images(vq):
    """5 grids of 64 x 64 codes: 4 images per pass at 512 x 512, so two passes; each image must have the bits it has
    when decoded alone."""
    m, vqvae = vq["model"], vq["vqvae"]
    codes = torch.randint(0, 8192, (5, 64, 64), generator=torch.Generator().manual_seed(22)).cuda()
    with torch.no_grad():
        both = vqvae.code2img(m, codes)
        single = torch.cat([vqvae.code2img(m, codes[i:i + 1]) for i in range(5)])
    assert both.shape == (5, 3, 512, 512)
    assert torch.equal(both, single)


# ----------------------------------------------------------------------------------------------------
# generate.super_resolution end to end
# ----------------------------------------------------------------------------------------------------
N_TXT = 101          # small text vocabulary: 8192 image codes + 101 text pieces + 27 command tokens = 8320


def _sr_model():
    from cogview_b200.model import GPT2Model
    cfg = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=256, num_attention_heads=4,
               max_sequence_length=1089)
    m = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                  num_attention_heads=cfg["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=1089,
                  max_memory_length=1345, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(seed=31, **cfg))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    return m


def test_super_resolution_end_to_end(vq, monkeypatch):
    """[ROI1] text [BASE] [BOI1] <1024 codes> -> nine magnify windows of up to 1293 tokens each (position ids wrap
    after [ROI2]; the K|V cache grows past 1089) -> 4096 codes -> one 512 x 512 image.  Greedy (top-k 1): the run with
    the sampling tail inside the decode graph gives the same tokens as the per-token host loop."""
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    tok = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", tok)
    m, vqvae = _sr_model(), vq["vqvae"]
    g = torch.Generator().manual_seed(23)
    text = (8192 + torch.randint(0, N_TXT, (6,), generator=g)).tolist()
    src = torch.randint(0, 8192, (1024,), generator=g).tolist()
    seq = torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['super-resolution'], [text, src], tokenizer=tok),
                       dtype=torch.long, device="cuda")

    class A:
        temperature, top_k, top_p, is_sparse = 1.0, 1, 0.0, 0
        img_tokenizer_num_tokens = 8192

    monkeypatch.setenv("COGVIEW_B200_GRAPH_SAMPLING", "1")
    torch.manual_seed(0)
    codes, imgs = generate.super_resolution(m, vq["model"], A, seq)
    assert codes.shape == (1, 4096) and imgs.shape == (1, 3, 512, 512)
    assert int(codes.min()) >= 0 and int(codes.max()) < 8192
    with torch.no_grad():
        assert torch.equal(imgs, vqvae.code2img(vq["model"], codes.view(1, 64, 64)))

    monkeypatch.setenv("COGVIEW_B200_GRAPH_SAMPLING", "0")
    torch.manual_seed(0)
    codes_eager, imgs_dbg = generate.super_resolution(m, vq["model"], A, seq, debug=True)
    agree = (codes_eager == codes).float().mean().item()
    print("super-resolution: graph sampling vs host loop token agreement %.4f" % agree)
    assert torch.equal(codes_eager, codes)
    assert imgs_dbg.shape == (2, 3, 512, 512)
    with torch.no_grad():
        src_img = vqvae.code2img(vq["model"], torch.tensor(src, device="cuda").view(1, 32, 32))
    assert torch.equal(imgs_dbg[:1], F.interpolate(src_img, size=(512, 512)))
    assert torch.equal(imgs_dbg[1:], imgs)
