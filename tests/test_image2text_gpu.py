"""GPU tests of image captioning (image2text): cv_attn_decode_shared (rows in groups that share a prompt's K|V), the
DecodeRunner's shared mode, and generate.image2text end to end.

Tolerances follow test_caption_batch_gpu.py: the kernel against a float64 softmax over each row's keys, to one bf16
rounding of the output (2^-8 relative) plus 1e-3 absolute; a shared-mode decode step against a uniform-mode step on a
cache holding each group's prefix in its rows, to 1e-2 of the logit scale and 2e-2 for the appended K|V; greedy tokens
equal a solo filling_sequence run up to the first position whose top-2 margin over the text vocabulary is within twice
that bound (the abs-max LayerNorm scales of the batch prompt forward and of the decode step are taken over the batch).
"""
import pytest
import torch

from oracle import recipes

pytestmark = pytest.mark.gpu

HD = 64


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import ops as _ops
    return _ops


# ----------------------------------------------------------------------------------------------------
# 1. cv_attn_decode_shared
# ----------------------------------------------------------------------------------------------------
# (groups, G, P, s, s_max, nsplit, heads): every value of each parameter appears, not the full product
KERNEL_CASES = [
    (1, 1, 1, 0, 24, 1, 4),
    (3, 2, 63, 1, 24, 3, 40),
    (8, 8, 64, 19, 24, 16, 4),
    (1, 16, 1028, 23, 24, 3, 40),
    (3, 17, 1300, 19, 24, 16, 4),
    (1, 64, 1028, 19, 24, 16, 40),
    (8, 8, 1028, 10, 24, 1, 40),
    (3, 64, 63, 0, 24, 1, 4),
    (1, 8, 64, 159, 160, 3, 4),          # more suffix keys than one pass of the combine kernel scores
]


@pytest.mark.parametrize("groups,G,P,s,s_max,nsplit,heads", KERNEL_CASES)
def test_attn_decode_shared(ops, groups, G, P, s, s_max, nsplit, heads):
    b, h = groups * G, heads * HD
    max_len = P + 7
    seed = groups * 100000 + G * 1000 + P + s + nsplit + heads
    gd = torch.Generator(device="cuda").manual_seed(seed)
    prefix = torch.randn((groups, max_len, 2 * h), generator=gd, device="cuda").to(torch.bfloat16)
    prefix[:, P:] = float("nan")                                  # past the prompt: never read
    suffix = torch.randn((b, s_max, 2 * h), generator=gd, device="cuda").to(torch.bfloat16)
    suffix[:, s:] = float("nan")                                  # slot s is written, the rest never touched
    qkv = torch.randn((b, 3 * h), generator=gd, device="cuda").to(torch.bfloat16)
    p0, s0 = prefix.clone(), suffix.clone()
    if nsplit == 3:                                               # the suffix length from the host
        out = ops.attn_decode_shared(qkv, prefix, suffix, heads, P, s=s, nsplit=nsplit)
    else:
        s_dev = torch.tensor([s], dtype=torch.int32, device="cuda")
        out = ops.attn_decode_shared(qkv, prefix, suffix, heads, P, s_dev=s_dev, nsplit=nsplit)
    torch.cuda.synchronize()
    q = qkv[:, :h].double().view(b, heads, HD)
    k_new, v_new = qkv[:, h:2 * h], qkv[:, 2 * h:]
    for r in range(b):
        g = r // G
        k = torch.cat((p0[g, :P, :h], s0[r, :s, :h], k_new[r:r + 1])).double().view(-1, heads, HD)
        v = torch.cat((p0[g, :P, h:], s0[r, :s, h:], v_new[r:r + 1])).double().view(-1, heads, HD)
        pr = torch.softmax(torch.einsum("hd,khd->hk", q[r], k) / HD ** 0.5, dim=-1)
        ref = torch.einsum("hk,khd->hd", pr, v).reshape(h)
        err = (out[r].double() - ref).abs()
        assert bool((err <= 2.0 ** -8 * ref.abs() + 1e-3).all()), (r, err.max().item())
    want = s0.clone()
    want[:, s, :h], want[:, s, h:] = k_new, v_new
    assert torch.equal(suffix.view(torch.int16), want.view(torch.int16))
    assert torch.equal(prefix.view(torch.int16), p0.view(torch.int16))


def test_attn_decode_shared_argument_errors(ops):
    from cogview_b200._lib import CogViewB200Error
    lib = ops.lib()
    heads, h = 4, 4 * HD
    qkv = torch.zeros((8, 3 * h), dtype=torch.bfloat16, device="cuda")
    prefix = torch.zeros((2, 40, 2 * h), dtype=torch.bfloat16, device="cuda")
    suffix = torch.zeros((8, 10, 2 * h), dtype=torch.bfloat16, device="cuda")
    out = torch.zeros((8, h), dtype=torch.bfloat16, device="cuda")
    ws = torch.zeros(lib.cv_attn_shared_workspace_bytes(8, heads, 64) // 4 + 4, dtype=torch.float32, device="cuda")
    base = dict(qkv=qkv.data_ptr(), prefix=prefix.data_ptr(), pbs=prefix.stride(0), P=30, max_len=40,
                suffix=suffix.data_ptr(), sbs=suffix.stride(0), s=3, s_max=10, out=out.data_ptr(), ws=ws.data_ptr(),
                b=8, groups=2, heads=heads, hd=HD, nsplit=2)

    def call(**kw):
        a = dict(base, **kw)
        rc = lib.cv_attn_decode_shared(a["qkv"], a["prefix"], a["pbs"], a["P"], a["max_len"], a["suffix"], a["sbs"],
                                       None, a["s"], a["s_max"], a["out"], a["ws"], a["b"], a["groups"], a["heads"],
                                       a["hd"], a["nsplit"], torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return rc
    assert call() == 0
    for kw in (dict(hd=32), dict(b=65, groups=1), dict(b=8, groups=3), dict(b=0), dict(P=41), dict(s=10),
               dict(s=-1), dict(nsplit=0), dict(nsplit=65), dict(qkv=qkv.data_ptr() + 2),
               dict(suffix=suffix.data_ptr() + 2), dict(prefix=prefix.data_ptr() + 2), dict(out=out.data_ptr() + 2),
               dict(pbs=prefix.stride(0) - 8), dict(sbs=suffix.stride(0) - 8)):
        assert call(**kw) < 0, kw
    with pytest.raises(CogViewB200Error):                         # through the wrapper: 8 rows in 3 groups
        ops.attn_decode_shared(qkv, torch.zeros((3, 40, 2 * h), dtype=torch.bfloat16, device="cuda"), suffix, heads,
                               30, s=3)
    with pytest.raises(CogViewB200Error):                         # s >= s_max
        ops.attn_decode_shared(qkv, prefix, suffix, heads, 30, s=10)


# ----------------------------------------------------------------------------------------------------
# 2. the shared-mode decode step
# ----------------------------------------------------------------------------------------------------
N_TXT = 101
CFG_TINY = dict(num_layers=2, vocab_size=58240, hidden_size=256, num_attention_heads=4)
CFG_4B_WIDTH = dict(num_layers=2, vocab_size=58240, hidden_size=2560, num_attention_heads=40)
CFG_GEN = dict(num_layers=2, vocab_size=8192 + N_TXT + 27, hidden_size=256, num_attention_heads=4)


def _model(cfg, maxlen, seed=7):
    from cogview_b200.model import GPT2Model
    m = GPT2Model(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                  num_attention_heads=cfg["num_attention_heads"], embedding_dropout_prob=0.0,
                  attention_dropout_prob=0.0, output_dropout_prob=0.0, max_sequence_length=maxlen,
                  max_memory_length=maxlen, checkpoint_activations=False)
    m.load_state_dict(recipes.gpt2_state_dict(num_layers=cfg["num_layers"], vocab_size=cfg["vocab_size"],
                                              hidden_size=cfg["hidden_size"], max_sequence_length=maxlen, seed=seed))
    m = m.cuda().bfloat16().eval()
    m.transformer.mems_mode = "kv"
    return m


@pytest.mark.parametrize("cfg,groups,G,P,s0", [(CFG_TINY, 3, 4, 100, 5), (CFG_TINY, 2, 17, 70, 0),
                                               (CFG_4B_WIDTH, 8, 8, 1028, 10)])
def test_shared_step_matches_a_uniform_step(ops, cfg, groups, G, P, s0):
    from cogview_b200.mpu import kv_cache
    from cogview_b200.mpu.decode import DecodeRunner
    model = _model(cfg, P + s0 + 8)
    tr = model.transformer
    b, run, dev = groups * G, s0 + 3, torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(b + P)
    pre = kv_cache._Caches(tr, groups, dev)
    pre.buf.copy_((torch.randn(pre.buf.shape, generator=g, device="cuda") * 0.5).to(torch.bfloat16))
    suf = kv_cache._SharedCaches(tr, b, groups, run, dev)
    suf.buf.copy_((torch.randn(suf.buf.shape, generator=g, device="cuda") * 0.5).to(torch.bfloat16))
    suf.prefix, suf.P = pre, P
    suf_eager = kv_cache._SharedCaches(tr, b, groups, run, dev)
    suf_eager.buf.copy_(suf.buf)
    suf_eager.prefix, suf_eager.P = pre, P
    pre_bits = pre.buf.clone()
    uni = kv_cache._Caches(tr, b, dev)
    for r in range(b):                                            # each group's prefix copied into its G rows
        uni.buf[:, r, :P] = pre.buf[:, r // G, :P]
        uni.buf[:, r, P:P + s0] = suf.buf[:, r, :s0]
    shared = DecodeRunner(model, suf, use_graph=True)
    eager = DecodeRunner(model, suf_eager, use_graph=False)
    uniform = DecodeRunner(model, uni, use_graph=True)
    assert shared.shared and not uniform.shared
    ids = torch.randint(0, 8192, (b, 1), generator=torch.Generator().manual_seed(1)).cuda()
    pos = torch.full((b, 1), P + s0, dtype=torch.long, device="cuda")
    with torch.no_grad():
        for step in range(3):
            ls = shared.step(ids, pos + step, s0 + step).clone()
            le = eager.step(ids, pos + step, s0 + step).clone()
            assert torch.equal(ls, le)                            # graph replay == per-operation launches
            lu = uniform.step(ids, pos + step, P + s0 + step).clone()
            scale = lu.abs().max().item()
            err = (ls - lu).abs().max().item()
            print("h=%d groups=%d G=%d P=%d step %d: logits max|diff| %.3e (scale %.3e)"
                  % (tr.hidden_size, groups, G, P, step, err, scale))
            assert err < 1e-2 * scale
            for i in range(cfg["num_layers"]):
                kp, ku = suf.buf[i, :, s0 + step].float(), uni.buf[i, :, P + s0 + step].float()
                assert (kp - ku).abs().max().item() < 2e-2 * ku.abs().max().item()
            ids = ls[:, :8192].argmax(-1, keepdim=True)
    assert shared.replays == 3 and torch.equal(suf.buf, suf_eager.buf)
    assert torch.equal(pre.buf.view(torch.int16), pre_bits.view(torch.int16))


# ----------------------------------------------------------------------------------------------------
# 3. image2text end to end
# ----------------------------------------------------------------------------------------------------
class _Args:
    temperature, top_k, top_p, is_sparse = 1.0, 1, 0.0, 0
    img_tokenizer_num_tokens = 8192
    max_inference_batch_size = 64


@pytest.fixture(scope="module")
def gen_model():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return _model(CFG_GEN, 1100, seed=31)


@pytest.fixture(scope="module")
def vq():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from cogview_b200 import vqvae
    model = vqvae.new_model()
    model.load_state_dict(recipes.vqvae_state_dict(seed=0))
    return model.cuda().eval()


@pytest.fixture
def tok(monkeypatch):
    from cogview_b200.generation import sampling
    t = sampling.TokenLayout(img_tokens=8192, txt_tokens=N_TXT)
    monkeypatch.setattr(sampling, "_TOKENIZER", t)
    return t


def _images(n, seed=0):
    from cogview_b200.vqvae.api import IMG_MEAN, IMG_STD
    g = torch.Generator().manual_seed(seed)
    img = torch.rand((n, 3, 256, 256), generator=g)
    img = (img - torch.tensor(IMG_MEAN).view(1, 3, 1, 1)) / torch.tensor(IMG_STD).view(1, 3, 1, 1)
    return img.cuda()


def _decisive_prefix(model, row, C):
    """Number of leading tokens of `row` whose choice had a top-2 margin over the text vocabulary (teacher-forced
    forward) above 2 x 1e-2 of the logit scale; the context always counts.  The first draw is checked too: it comes
    from a forward at the batch of all images, whose LayerNorm scales differ from the solo forward's."""
    s = row.shape[0]
    with torch.no_grad():
        lg, *_ = model(row[:-1].view(1, -1), torch.arange(s - 1, device="cuda").view(1, -1),
                       torch.tril(torch.ones((1, 1, s - 1, s - 1), device="cuda")), None, None, 0)
    lg = lg[0, C - 1:, 8192:8192 + N_TXT].float()                # predicts tokens C ..
    top = lg.topk(2, dim=-1).values
    margin = top[:, 0] - top[:, 1]
    bad = (margin <= 2 * 1e-2 * lg.abs().amax(-1)).nonzero()
    return C + (int(bad[0]) if bad.numel() else s - C)


def _fresh_pool(model):
    model.transformer._kv_pool = {}
    model.transformer._kv = None


@pytest.mark.parametrize("n,num,mbz", [(1, 8, 64), (3, 4, 64), (8, 8, 64), (3, 1, 64), (2, 16, 8)])
def test_greedy_captions_follow_each_image_alone(gen_model, vq, tok, n, num, mbz):
    from cogview_b200 import generate, vqvae
    from cogview_b200.generation import sampling

    class A(_Args):
        max_inference_batch_size = mbz
    imgs = _images(n, seed=n * 10 + num)
    _fresh_pool(gen_model)
    out = generate.image2text(gen_model, vq, A, imgs, num=num)
    pool = gen_model.transformer._kv_pool
    nb = min(num, mbz)
    per = max(1, mbz // nb)
    assert ('shared', min(n, per) * nb, min(n, per), 19) in pool  # the shared route ran
    assert all(k <= per for k in pool if isinstance(k, int))      # no cache of a row per beam
    codes = vqvae.img2code(vq, imgs)
    checked = 0
    for (rows, captions), c in zip(out, codes):
        seq = torch.tensor(generate.build_query(generate.QUERY_TEMPLATES['image2text'], [c.tolist()], tok),
                           dtype=torch.long, device="cuda")
        sampling.add_interlacing_beam_marks(seq, nb=nb)
        with torch.no_grad():
            solo = sampling.filling_sequence(gen_model, seq, A)
        assert rows.shape == (num, 1048) and len(captions) == num
        k = _decisive_prefix(gen_model, solo[0], 1028)
        assert torch.equal(rows[:, :k], solo[:1, :k].expand(num, -1)), k
        assert captions == [(r[1028:] - 8192).tolist() for r in rows]
        checked += k - 1028
    print("n=%d num=%d: %d generated tokens compared" % (n, num, checked))
    assert checked > 0


def test_top_k_sampling_gives_text_ids_and_repeats_with_the_seed(gen_model, vq, tok):
    from cogview_b200 import generate

    class A(_Args):
        top_k = 200
    imgs = _images(8, seed=5)
    _fresh_pool(gen_model)
    torch.manual_seed(3)
    out = generate.image2text(gen_model, vq, A, imgs, num=8)
    pool = gen_model.transformer._kv_pool
    assert 64 not in pool and set(pool) == {8, ('shared', 64, 8, 19)}
    for rows, captions in out:
        gen = rows[:, 1028:]
        assert int(gen.min()) >= 8192 and int(gen.max()) < 8192 + N_TXT
        assert all(0 <= x < N_TXT for cap in captions for x in cap)
        assert len({tuple(r.tolist()) for r in gen}) > 1
    torch.manual_seed(3)
    again = generate.image2text(gen_model, vq, A, imgs, num=8)
    assert all(a[1] == b[1] for a, b in zip(out, again))


def test_text2image_and_image2text_runs_do_not_disturb_each_other(gen_model, vq, tok):
    from cogview_b200 import generate
    from cogview_b200.generation import sampling
    g = torch.Generator().manual_seed(4)
    caps = []
    for n in (5, 17, 40):
        text = (8192 + torch.randint(0, N_TXT, (n,), generator=g)).tolist()
        caps.append(torch.tensor([tok['[ROI1]']] + text + [tok['[BASE]'], tok['[BOI1]']] + [-4] * 40,
                                 dtype=torch.long, device="cuda"))
    imgs = _images(3, seed=8)

    def t2i():
        torch.manual_seed(1)
        with torch.no_grad():
            return sampling.filling_sequences(gen_model, caps, _Args)

    def i2t():
        torch.manual_seed(2)
        return [r for r, _ in generate.image2text(gen_model, vq, _Args, imgs, num=4)]
    _fresh_pool(gen_model)
    t_alone = t2i()
    _fresh_pool(gen_model)
    i_alone = i2t()
    t_after = t2i()
    i_after = i2t()
    assert all(torch.equal(a, b) for a, b in zip(t_alone, t_after))
    assert all(torch.equal(a, b) for a, b in zip(i_alone, i_after))
