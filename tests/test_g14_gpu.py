"""ViT-g-14 and ViT-bigG-14 on the GPU: attention at head dims 88 and 104 (HD % 16 == 8: an 8-wide tail in QK^T and
P.V, and a Q fragment whose upper half must not be loaded), the embed kernels at the new widths, the towers against the
float64 oracle of tower_ref.py and an independent transformers golden, the full-depth synthetic towers against the
fp32 oracle, and the drop-in paths (load_clip, ClipMapper, B200KnnService) at bigG's sizes."""
import os

import numpy as np
import pytest

import test_tower_parity_gpu as TP
import tower_ref as R
from oracle import clip_ref
from test_embed_gpu import assert_attention_close, attention_ref64, run_attention
from test_g14_cpu import g14_cases, g14_state_dict
from test_mclip_gpu import run_attention_len

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3
HDS = (88, 104)
# the longest T the whole-K/V kernel takes: 2 * ceil32(T) * (hd + 16) * 2 bytes <= 200 KB
LONGEST_WHOLE = {88: 480, 104: 416}


def _qkv(B, T, w, seed, device="cuda"):
    import torch

    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(B * T, 3 * w, device=device, generator=g).bfloat16()


# ---- attention ----------------------------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("hd", HDS)
def test_attention_matches_float64(hd, causal):
    """Three heads (the last head's next columns are K) at every T around the 16-row query blocks and 32-key blocks,
    the real image T of 257, both sides of the whole-K/V / streaming switch and a long streamed T."""
    heads, B = 3, 2
    w = heads * hd
    top = LONGEST_WHOLE[hd]
    for T in (1, 17, 31, 32, 33, 63, 64, 65, 257, top, top + 1, top + 65, 730):
        qkv = _qkv(B, T, w, 11 * T + hd + causal)
        out = run_attention(qkv, B, T, heads, w, causal)
        ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
        assert_attention_close(out, ref, bound, "hd=%d T=%d causal=%d" % (hd, T, causal))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("T", [257, 730])
@pytest.mark.parametrize("hd", HDS)
def test_attention_per_sample_lengths(hd, T):
    """Key lengths through b200_attention_len_bf16_device, on the whole-K/V kernel (T 257) and the streaming kernel
    (T 730): each sample attends to its own keys, and its rows past the length are exactly zero."""
    heads = 2
    w = heads * hd
    lengths = sorted({1, 2, 31, 32, 33, 127, 128, 129, T - 1, T} & set(range(1, T + 1)))
    B = len(lengths)
    qkv = _qkv(B, T, w, 4242 + hd + T)
    out = run_attention_len(qkv, lengths, B, T, heads, w).view(B, T, w)
    for b, L in enumerate(lengths):
        src = qkv.view(B, T, 3 * w)[b, :L].contiguous()
        ref, bound, _ = attention_ref64(src, 1, L, heads, hd, 0)
        assert_attention_close(out[b, :L], ref, bound, "hd=%d T=%d len=%d" % (hd, T, L))
        assert bool((out[b, L:] == 0).all()), "len=%d: rows past the length are not zero" % L


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("hd", HDS)
@pytest.mark.parametrize("T", [65, 257, 481])
def test_attention_one_hot_v_probes(T, hd, causal):
    """V is zero except one 1.0 per (sample, head) at key t, dim j, with j in {0, 7, 8, HD-9, HD-8, HD-1}: the 8-wide
    tail's n8 tile and the tiles around it.  That output dim is P[r, t] alone, every other output is exactly 0."""
    import torch

    keys = sorted({t for t in (0, 1, 31, 32, 63, 64, 65, T - 1) if t < T})
    dims = [0, 7, 8, hd - 9, hd - 8, hd - 1]
    B, heads = 6, len(keys)
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(T + hd + causal)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = qkv.view(B, T, 3, heads, hd)
    view[:, :, 2] = 0.0
    probe = {}
    for h, t in enumerate(keys):
        for b in range(B):
            j = dims[(b + h) % len(dims)]
            view[b, t, 2, h, j] = 1.0
            probe[(b, h)] = (t, j)
    qkv = qkv.bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal).view(B, T, heads, hd).double()
    _, _, P = attention_ref64(qkv, B, T, heads, hd, causal)
    want = torch.zeros(B, T, heads, hd, dtype=torch.float64, device="cuda")
    for (b, h), (t, j) in probe.items():
        want[b, :, h, j] = P[b, h, :, t]
    zero = want == 0
    assert bool((out[zero] == 0).all()), "%d outputs that must be exactly 0 are not (first: %s)" % (
        int((out[zero] != 0).sum()), torch.nonzero(zero & (out != 0))[:1].tolist())
    err = (out[~zero] - want[~zero]).abs()
    assert bool((err <= (2.0 ** -7 + 2.0 ** -12) * want[~zero]).all()), \
        "probe P[r, t]: max rel err %g" % (err / want[~zero]).max().item()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("hd", HDS)
@pytest.mark.parametrize("T", [77, 257, 481])
def test_attention_tail_only_scores(T, hd, causal):
    """Q and K are zero outside dims HD-8..HD-1, so the scores come from the 8-wide QK^T tail alone: a kernel that
    drops it sees all-zero scores and returns the uniform average of V, far outside the bound."""
    import torch

    heads, B = 3, 2
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(T * 5 + hd + causal)
    x = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = x.view(B, T, 3, heads, hd)
    view[:, :, :2, :, :hd - 8] = 0.0
    view[:, :, :2, :, hd - 8:] *= 3.0
    qkv = x.bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal)
    ref, bound, P = attention_ref64(qkv, B, T, heads, hd, causal)
    assert_attention_close(out, ref, bound, "tail only hd=%d T=%d causal=%d" % (hd, T, causal))
    # the scores are far from uniform, so the uniform average is far outside the bound
    v = qkv.double().view(B, T, 3, heads, hd)[:, :, 2]
    if causal:
        uniform = v.cumsum(1) / torch.arange(1, T + 1, device="cuda", dtype=torch.float64)[None, :, None, None]
    else:
        uniform = v.mean(1, keepdim=True).expand(B, T, heads, hd)
    uniform = uniform.reshape(B * T, w)
    assert float(((uniform - ref).abs() / bound).max()) > 10.0


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("hd", HDS)
@pytest.mark.parametrize("T", [257, 481])
def test_attention_next_head_does_not_leak(T, hd, causal):
    """The 8 qkv columns after each head's Q (head h + 1's Q dims 0..7; K dims 0..7 of head 0 after the last head) are
    +-1e4.  They take no part in any head's true scores (the K dims they meet are zero, and head 0's Q dims 0..7 are
    zero), so the float64 reference is an ordinary attention; a kernel that loads them into the zero half of the last
    Q fragment multiplies them by K padding or K dims and its scores explode."""
    import torch

    heads, B = 3, 2
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(T * 7 + hd + causal)
    x = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = x.view(B, T, 3, heads, hd)
    sign = torch.where(torch.rand(B, T, heads, 8, device="cuda", generator=g) < 0.5, -1e4, 1e4)
    view[:, :, 0, :, :8] = sign
    view[:, :, 0, 0, :8] = 0.0            # head 0's Q dims 0..7 meet the +-1e4 of K head 0
    view[:, :, 1, :, :8] = 0.0            # the K dims every other head's +-1e4 Q dims meet
    view[:, :, 1, 0, :8] = sign[:, :, 0]  # after the last head's Q: K of head 0
    qkv = x.bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal)
    ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
    assert_attention_close(out, ref, bound, "next-head leak hd=%d T=%d causal=%d" % (hd, T, causal))


# ---- kernels at the new widths ------------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("w", [1408, 1664])
def test_layernorm_at_g14_widths(w):
    """Both LayerNorm entries at the image widths, at 256 x 257 rows (above the persistent grid's 6336 warps)."""
    from test_embed_kernels_gpu import check_layernorm

    check_layernorm(w, 256 * 257, ((1e-5, None), (1e-5, 1e-5)))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("w,D,T", [(1408, 1024, 257), (1664, 1280, 257), (1280, 1280, 77)])
@pytest.mark.parametrize("B", [1, 3, 1024])
def test_pool_ln_proj_at_g14_shapes(w, D, T, B):
    from test_embed_kernels_gpu import test_pool_ln_proj_matches_float64

    test_pool_ln_proj_matches_float64(w, D, T, B)


@pytest.mark.timeout(120)
def test_text_embed_at_bigG_width():
    from test_embed_kernels_gpu import test_text_embed_bit_exact

    test_text_embed_bit_exact(1280, 77, 49408)


# ---- tower parity (tower_ref.py) at LAYERS = 2 ---------------------------------------------------------------------------

class G14Case(TP.Case):
    """test_tower_parity_gpu.Case for a g14_cases() entry: the same checks, over this file's cases."""

    def __init__(self, name, weights):
        self.name, self.weights = name, weights
        self.label = "%s/%s" % (name, weights)
        self.arch = g14_cases()[name]
        self.sd = g14_state_dict(name, weights)
        self.W = R.handle_weights(self.sd, "cuda")
        self.models = {}
        self.worst = {}


CASES = [(n, w) for n in g14_cases() for w in R.WEIGHTS]


@pytest.fixture(scope="module", params=CASES, ids=["%s-%s" % c for c in CASES])
def case(request):
    import torch

    c = G14Case(*request.param)
    yield c
    c.report()
    c.envelope.cache_clear()
    del c.models, c.W
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.mark.timeout(600)
def test_tower_batch1_graph_path(case):
    TP.test_batch1_graph_path(case)


@pytest.mark.timeout(600)
def test_tower_chunk_seams_and_entries(case):
    TP.test_chunk_seams_and_entries(case)


@pytest.mark.timeout(600)
def test_tower_large_batch_wide_gemm(case):
    TP.test_large_batch_wide_gemm(case)


# ---- an independent golden: transformers CLIPModel at head dims 104 (vision) and 88 (text) ------------------------------

def _load_golden_generator():
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_g14_golden", os.path.join(GOLDEN, "make_g14_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.timeout(300)
def test_tiny_g14_matches_hf_golden_and_oracle():
    from test_embed_gpu import _arch

    import clip_retrieval_b200 as m

    gen = _load_golden_generator()
    cfg, n = gen.CFG, gen.N
    assert cfg.vision.width // cfg.vision.heads == 104 and cfg.text.width // cfg.text.heads == 88
    sd = clip_ref.make_state_dict(cfg, seed=0)
    model = m.B200Clip(_arch(m, cfg), device=0, max_batch=2).load_state_dict(sd)
    px = clip_ref.synth_images(n, cfg, seed=0)
    tk = clip_ref.synth_tokens(n, cfg, seed=0)
    gold = np.load(gen.OUT)
    fi = model.encode_image(px.cuda()).cpu().numpy()
    ft = model.encode_text(tk.cuda()).cpu().numpy()
    for got, ref_hf, ref_or in ((fi, gold["image_features"], clip_ref.encode_image(sd, cfg, px).numpy()),
                                (ft, gold["text_features"], clip_ref.encode_text(sd, cfg, tk).numpy())):
        assert (1 - clip_ref.cosine(got, ref_hf)).max() <= COS_TOL, 1 - clip_ref.cosine(got, ref_hf)
        assert (1 - clip_ref.cosine(got, ref_or)).max() <= COS_TOL
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), np.linalg.norm(ref_or, axis=1), rtol=2e-2)
    assert np.array_equal(model.embed_image_device(px.cuda()).cpu().numpy(), model.embed_image(px))


# ---- full-depth synthetic towers ---------------------------------------------------------------------------------------

@pytest.mark.timeout(1800)
@pytest.mark.parametrize("key", ["open_clip:ViT-g-14", "open_clip:ViT-bigG-14"])
def test_full_depth_tower_matches_fp32_oracle(key):
    """Every layer at the real sizes, 2 samples: 1 - cos <= 1e-3 and norms within 2 % of the fp32 oracle (the image
    oracle runs on the GPU in fp32 without TF32, the text oracle on the host); host entry = device entry bit for bit."""
    import torch

    import clip_retrieval_b200 as m

    torch.set_num_threads(max(1, os.cpu_count() or 1))
    a = m.G14_ARCHS[key]
    cfg = R.clip_cfg(a)
    sd = clip_ref.make_state_dict(cfg, seed=0)
    model = m.B200Clip(a, device=0, max_batch=2).load_state_dict(sd)
    px = clip_ref.synth_images(2, cfg, seed=1)
    tk = clip_ref.synth_tokens(2, cfg, seed=1)
    fi = model.encode_image(px.cuda()).cpu().numpy()
    ft = model.encode_text(tk.cuda()).cpu().numpy()
    ei, et = model.embed_image(px), model.embed_text(tk)
    assert np.array_equal(model.embed_image_device(px.cuda()).cpu().numpy(), ei)
    assert np.array_equal(model.embed_text_device(tk.cuda()).cpu().numpy(), et)
    del model
    torch.cuda.empty_cache()
    ref_t = clip_ref.encode_text(sd, cfg, tk).numpy()
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        sd_dev = {k: v.cuda() for k, v in sd.items() if k.startswith("visual.")}
        ref_i = clip_ref.encode_image(sd_dev, cfg, px.cuda()).cpu().numpy()
        del sd_dev
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
        torch.cuda.empty_cache()
    for what, got, ref in (("image", fi, ref_i), ("text", ft, ref_t)):
        d = 1 - clip_ref.cosine(got, ref)
        print("\n%s %s full depth: 1 - cos %s" % (key, what, d))
        assert d.max() <= COS_TOL, (what, d)
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), np.linalg.norm(ref, axis=1), rtol=2e-2)
    for what, got, ref in (("image", ei, ref_i), ("text", et, ref_t)):
        n = ref / np.linalg.norm(ref, axis=1, keepdims=True)
        assert (1 - clip_ref.cosine(got, n)).max() <= COS_TOL, what


# ---- drop-in paths ------------------------------------------------------------------------------------------------------

BIGG = "synthetic:open_clip:ViT-bigG-14/laion2b_s39b_b160k"


@pytest.mark.timeout(1200)
def test_bigG_load_clip_mapper_and_service():
    """load_clip of the synthetic bigG, a ClipMapper batch and a ragged last batch (the same rows as the first batch's
    head, bit for bit), and one text query through B200KnnService against a d = 1280 flat index."""
    import torch

    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import SimpleTokenizer
    from oracle import synth_ref

    # the arguments ClipMapper passes, so that both share one cached handle as the reference's builders do
    model, _, _ = m.load_clip(clip_model=BIGG, use_jit=False, warmup_batch_size=4, clip_cache_path=None)
    assert model.arch == m.G14_ARCHS["open_clip:ViT-bigG-14"] and model.max_batch == 4
    mapper = m.ClipMapper(True, True, False, False, BIGG, False, "", warmup_batch_size=4)
    assert mapper.model is model
    a = model.arch
    px = clip_ref.synth_images(5, R.clip_cfg(a), seed=3)
    tk = clip_ref.synth_tokens(5, R.clip_cfg(a), seed=3)
    full = mapper({"image_tensor": px[:4], "text_tokens": tk[:4], "image_filename": list("abcd"), "text": list("abcd")})
    last = mapper({"image_tensor": px[4:], "text_tokens": tk[4:], "image_filename": ["e"], "text": ["e"]})
    for k in ("image_embs", "text_embs"):
        assert full[k].dtype == np.float16 and full[k].shape == (4, 1280) and last[k].shape == (1, 1280)
        np.testing.assert_allclose(np.linalg.norm(full[k].astype(np.float32), axis=1), 1.0, atol=2e-3)
    one = mapper({"image_tensor": px[4:5], "text_tokens": tk[4:5], "image_filename": ["e"], "text": ["e"]})
    assert np.array_equal(one["image_embs"], last["image_embs"]) and np.array_equal(one["text_embs"], last["text_embs"])
    assert np.array_equal(model.embed_image_device(px[:4].cuda()).cpu().numpy(), full["image_embs"])

    d, n, k = a.embed_dim, 3000, 20
    X = synth_ref.rows_f16(n, d, seed=5)
    idx = m.B200FlatIndex(d)
    idx.add(X)
    tok = SimpleTokenizer(os.path.join(GOLDEN, "bpe_tiny.txt.gz"))
    res = m.ClipResource(model, tokenizer=tok, image_index=idx, text_index=idx)
    svc = m.B200KnnService({"bigG": res})
    got = svc.query(text_input="a photo of a cat", modality="image", num_images=k, num_result_ids=k, deduplicate=False)
    q = svc.compute_query_device(res, text_input="a photo of a cat")
    assert q.shape == (1, d) and abs(float(q.norm()) - 1.0) < 1e-3
    D, I = idx.search_device(q, k)
    assert [r["id"] for r in got] == [int(i) for i in I[0].cpu().numpy()]
    sims = np.array([r["similarity"] for r in got])
    assert len(got) == k and np.all(np.diff(sims) <= 1e-7)
    del svc, res, mapper, model
    m.load_clip.cache_clear()
    torch.cuda.empty_cache()
