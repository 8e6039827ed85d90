"""SigLIP on the GPU: attention at head dim 72 (the HD % 16 == 8 tail), the latent-query attention pool and the text
tail against float64, the towers against the fp32 oracle (tests/siglip_ref.py) and transformers' golden, the entry
points (graph replay, chunk seams, host vs device) and load_clip -> ClipMapper -> B200KnnService end to end."""
import os
from dataclasses import replace

import numpy as np
import pytest

import siglip_ref
from test_embed_gpu import assert_attention_close, attention_ref64, run_attention
from test_mclip_gpu import run_attention_len
from test_siglip_cpu import (captions, cos_dist, golden_module, sensitise, structured_images, tiny_arch,
                             tiny_tokenizer_json)

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3
HD = 72


def _qkv(B, T, w, seed):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()


# ---- attention at head dim 72 ---------------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
def test_attention_hd72_matches_float64(causal):
    """Three heads (the last head's next columns are K); T on both sides of the whole-K/V (T <= 576) / streaming
    switch, SO400M's 256 and 729 image tokens."""
    heads, B = 3, 2
    w = heads * HD
    for T in (1, 16, 17, 33, 64, 196, 256, 576, 577, 729, 1024):
        qkv = _qkv(B, T, w, 11 * T + causal)
        out = run_attention(qkv, B, T, heads, w, causal)
        ref, bound, _ = attention_ref64(qkv, B, T, heads, HD, causal)
        assert_attention_close(out, ref, bound, "hd=72 T=%d causal=%d" % (T, causal))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("T", [256, 729])
def test_attention_hd72_per_sample_lengths(T):
    heads = 2
    w = heads * HD
    lengths = sorted({1, 2, 31, 32, 33, 127, 128, 129, T - 1, T})
    B = len(lengths)
    qkv = _qkv(B, T, w, 4242 + T)
    out = run_attention_len(qkv, lengths, B, T, heads, w).view(B, T, w)
    for b, L in enumerate(lengths):
        src = qkv.view(B, T, 3 * w)[b, :L].contiguous()
        ref, bound, _ = attention_ref64(src, 1, L, heads, HD, 0)
        assert_attention_close(out[b, :L], ref, bound, "hd=72 T=%d len=%d" % (T, L))
        assert bool((out[b, L:] == 0).all())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T", [65, 256, 729])
def test_attention_hd72_one_hot_v_probes(T, causal):
    """V zero except one 1.0 per (sample, head) at key t, dim j in {0, 7, 8, 63, 64, 71}: that output dim is P[r, t]
    alone and every other output is exactly 0."""
    import torch

    keys = sorted({t for t in (0, 1, 31, 32, 63, 64, T - 1) if t < T})
    dims = [0, 7, 8, 63, 64, 71]
    B, heads = 6, len(keys)
    w = heads * HD
    g = torch.Generator(device="cuda").manual_seed(T + causal)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = qkv.view(B, T, 3, heads, HD)
    view[:, :, 2] = 0.0
    probe = {}
    for h, t in enumerate(keys):
        for b in range(B):
            j = dims[(b + h) % len(dims)]
            view[b, t, 2, h, j] = 1.0
            probe[(b, h)] = (t, j)
    qkv = qkv.bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal).view(B, T, heads, HD).double()
    _, _, P = attention_ref64(qkv, B, T, heads, HD, causal)
    want = torch.zeros(B, T, heads, HD, dtype=torch.float64, device="cuda")
    for (b, h), (t, j) in probe.items():
        want[b, :, h, j] = P[b, h, :, t]
    zero = want == 0
    assert bool((out[zero] == 0).all())
    err = (out[~zero] - want[~zero]).abs()
    assert bool((err <= (2.0 ** -7 + 2.0 ** -12) * want[~zero]).all())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T", [256, 729])
def test_attention_hd72_tail_only_scores_and_next_head(T, causal):
    """Scores from dims 64..71 alone (a kernel that drops the 8-wide tail returns the uniform average), then +-1e4 in
    the 8 columns after each head's Q (the next head's Q, or K): a kernel that reads past dim 71 is far off."""
    import torch

    heads, B = 3, 2
    w = heads * HD
    g = torch.Generator(device="cuda").manual_seed(T * 5 + causal)
    x = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = x.view(B, T, 3, heads, HD)
    view[:, :, :2, :, :HD - 8] = 0.0
    view[:, :, :2, :, HD - 8:] *= 3.0
    qkv = x.bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal)
    ref, bound, _ = attention_ref64(qkv, B, T, heads, HD, causal)
    assert_attention_close(out, ref, bound, "tail only T=%d causal=%d" % (T, causal))
    v = qkv.double().view(B, T, 3, heads, HD)[:, :, 2]
    uniform = (v.cumsum(1) / torch.arange(1, T + 1, device="cuda", dtype=torch.float64)[None, :, None, None]) if causal \
        else v.mean(1, keepdim=True).expand(B, T, heads, HD)
    assert float(((uniform.reshape(B * T, w) - ref).abs() / bound).max()) > 10.0

    y = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    qkv = y.bfloat16()
    ref, bound, _ = attention_ref64(qkv, B, T, heads, HD, causal)
    big = y.view(B, T, 3 * w).clone()
    for h in range(heads):
        big[:, :, (h + 1) * HD:(h + 1) * HD + 8] = 1e4 * torch.sign(torch.randn(B, T, 8, device="cuda", generator=g))
    # the 8 columns after head h's Q are head h + 1's Q (after the last head, K of head 0): the reference reads them
    # only where they belong, so a kernel whose Q tail reads dims 72..79 of a head scores against +-1e4
    big_bf = big.reshape(B * T, 3 * w).bfloat16()
    ref2, bound2, _ = attention_ref64(big_bf, B, T, heads, HD, causal)
    out2 = run_attention(big_bf, B, T, heads, w, causal)
    assert_attention_close(out2, ref2, bound2, "next-head columns T=%d causal=%d" % (T, causal))


# ---- latent-query attention pool --------------------------------------------------------------------------------------------

def run_latent_pool(kv, q, B, T, heads, w):
    import torch
    from clip_retrieval_b200._lib import lib, check

    out = torch.full((B, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    check(lib.b200_latent_pool_attention_device(kv.data_ptr(), B, T, heads, w, q.data_ptr(), out.data_ptr(), 0,
                                                torch.cuda.current_stream().cuda_stream), "latent_pool")
    torch.cuda.synchronize()
    return out


def latent_pool_ref64(kv, q, B, T, heads, hd):
    """float64 pool and its per-element bound.
    |out - ref| <= 2^-8 |ref| + (2 ds + (T + 2) 2^-22) * sum_t P_t |v_t|
    - 2^-8 |ref|: the bf16 store (half an ulp of 8 significant bits).
    - ds: the fp32 error of a score, hd 2^-24 * 2 * max_t |q| . |k_t| hd^-0.5 (hd fused multiply-adds in dim order); a
      score off by ds moves P_t by at most a factor exp(2 ds).
    - (T + 2) 2^-22: expf, the fp32 sums over T keys (l and P.V, each an ordered sum of non-negative weights) and the
      final division, each within a few ulps per step."""
    import torch

    w = heads * hd
    k = kv.double().view(B, T, 2, heads, hd)[:, :, 0].permute(0, 2, 1, 3)
    v = kv.double().view(B, T, 2, heads, hd)[:, :, 1].permute(0, 2, 1, 3)
    qh = q.double().view(heads, 1, hd)
    s = (qh @ k.transpose(-1, -2)) * hd ** -0.5          # [B, heads, 1, T]
    mag = (qh.abs() @ k.abs().transpose(-1, -2)) * hd ** -0.5
    P = torch.softmax(s, -1)
    ref = (P @ v).reshape(B, w)
    spread = (P @ v.abs()).reshape(B, w)
    ds = (hd * 2.0 ** -23 * mag.amax(-1)).expand(B, heads, hd).reshape(B, w)
    bound = 2.0 ** -8 * ref.abs() + (2 * ds + (T + 2) * 2.0 ** -22) * spread
    return ref, bound


@pytest.mark.timeout(300)
@pytest.mark.parametrize("hd", [64, 72])
def test_latent_pool_matches_float64(hd):
    import torch

    heads = 3
    w = heads * hd
    for T in (1, 16, 196, 256, 576, 729, 1024):
        for B in (1, 3, 256):
            g = torch.Generator(device="cuda").manual_seed(T * 7 + B + hd)
            kv = (torch.randn(B * T, 2 * w, device="cuda", generator=g) * 2).bfloat16()
            q = torch.randn(w, device="cuda", generator=g) * 2
            out = run_latent_pool(kv, q, B, T, heads, w).double()
            ref, bound = latent_pool_ref64(kv, q, B, T, heads, hd)
            err = (out - ref).abs()
            assert bool((err <= bound).all()), "hd=%d T=%d B=%d: worst err/bound %.3g" % (
                hd, T, B, float((err / bound).max()))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("hd", [64, 72])
def test_latent_pool_one_hot_key(hd):
    """K zero except key t* of each (sample, head), aligned with q: its score is ~300 above every other, whose weights
    are exactly 0.0 in fp32, so the output must equal v_{t*} bit for bit (a key counted twice, skipped or taken from
    the wrong sample or head shows)."""
    import torch

    heads, B = 2, 3
    w = heads * hd
    for T in (1, 16, 196, 729, 1024):
        g = torch.Generator(device="cuda").manual_seed(T + hd)
        q = torch.randn(w, device="cuda", generator=g)
        kv = torch.zeros(B, T, 2, heads, hd, device="cuda")
        kv[:, :, 1] = torch.randn(B, T, heads, hd, device="cuda", generator=g)
        for b in range(B):
            for h in range(heads):
                t = (b * 37 + h * 101 + T // 2) % T
                qh = q[h * hd:(h + 1) * hd]
                kv[b, t, 0, h] = qh * (300.0 * hd ** 0.5 / float(qh.dot(qh)))
        kv = kv.reshape(B * T, 2 * w).bfloat16()
        want = kv.view(B, T, 2, heads, hd)[:, :, 1].float()   # the bf16 values
        out = run_latent_pool(kv, q, B, T, heads, w)
        idx = [(b * 37 + h * 101 + T // 2) % T for b in range(B) for h in range(heads)]
        exp = torch.stack([torch.cat([want[b, idx[b * heads + h], h] for h in range(heads)]) for b in range(B)])
        assert torch.equal(out.float(), exp), "hd=%d T=%d" % (hd, T)


# ---- text tail ----------------------------------------------------------------------------------------------------------

@pytest.mark.timeout(120)
@pytest.mark.parametrize("w,D", [(768, 768), (1152, 1152), (144, 144)])
def test_text_tail_matches_float64(w, D):
    """LN(eps 1e-6) of row T - 1 and the biased projection, raw (fp32 feat) and normalised; a row whose variance is
    ~1e-6 makes eps 1e-5 vs 1e-6 visible."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    B, T = 5, 16
    g = torch.Generator(device="cuda").manual_seed(w)
    x = torch.randn(B * T, w, device="cuda", generator=g)
    x[T - 1] = 3.0 + 1e-3 * torch.randn(w, device="cuda", generator=g)     # sample 0's last row: variance 1e-6
    x = x.bfloat16()
    gam = 1 + 0.1 * torch.randn(w, device="cuda", generator=g)
    bet = 0.05 * torch.randn(w, device="cuda", generator=g)
    proj = (torch.randn(w, D, device="cuda", generator=g) * w ** -0.5).bfloat16()
    bias = 0.1 * torch.randn(D, device="cuda", generator=g)
    feat = torch.empty(B, D, device="cuda")
    out = torch.empty(B, D, device="cuda")
    check(lib.b200_pool_last_ln_proj_bias_device(x.data_ptr(), B, T, w, gam.data_ptr(), bet.data_ptr(), 1e-6,
                                                 proj.data_ptr(), bias.data_ptr(), D, feat.data_ptr(), out.data_ptr(),
                                                 0, 1, 0, torch.cuda.current_stream().cuda_stream), "text_tail")
    torch.cuda.synchronize()
    r = x.double().view(B, T, w)[:, -1]
    y = (r - r.mean(-1, keepdim=True)) / torch.sqrt(r.var(-1, unbiased=False, keepdim=True) + 1e-6)
    y = y * gam.double() + bet.double()
    ref = y @ proj.double() + bias.double()
    # fp32 LN (relative ~1e-6 of |y|) and w-term fp32 dot products
    tol = 1e-5 * (y.abs() @ proj.double().abs()) + 1e-6 * ref.abs() + 1e-6
    assert bool(((feat.double() - ref).abs() <= tol).all()), float(((feat.double() - ref).abs() / tol).max())
    nrm = ref / ref.norm(dim=-1, keepdim=True)
    assert float((out.double() - nrm).abs().max()) <= 1e-4


@pytest.mark.timeout(120)
def test_patch_gemm_no_class_row():
    """The SigLIP patch embedding on the GEMM entry: bias, positional rows as residual (res_row_mod = g^2, offset 0), no
    class-row gap; NaN sentinels past the rows it owns stay NaN."""
    import torch
    import clip_retrieval_b200._lib as L

    B, g2, w, K = 3, 196, 768, 768
    gen = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randn(B * g2, K, device="cuda", generator=gen).bfloat16()
    W = (torch.randn(w, K, device="cuda", generator=gen) * K ** -0.5).bfloat16()
    bias = 0.1 * torch.randn(w, device="cuda", generator=gen)
    pos = torch.randn(g2, w, device="cuda", generator=gen).bfloat16()
    C = torch.full((B * g2 + 7, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    ep = L.GemmEpilogueC(bias.data_ptr(), pos.data_ptr(), w, g2, 0, w, 0, 0, None, None, 0, None)
    L.check(L.lib.b200_gemm_bf16_ex_device(A.data_ptr(), W.data_ptr(), C.data_ptr(), B * g2, w, K, ep, 0, 0, 0,
                                           torch.cuda.current_stream().cuda_stream), "gemm")
    torch.cuda.synchronize()
    ref = A.double() @ W.double().t() + bias.double() + pos.double().repeat(B, 1)
    mag = A.double().abs() @ W.double().abs().t() + bias.double().abs() + pos.double().abs().repeat(B, 1)
    got = C[:B * g2].double()
    assert bool(((got - ref).abs() <= 2.0 ** -8 * ref.abs() + K * 2.0 ** -23 * mag + 1e-6).all())
    assert bool(torch.isnan(C[B * g2:].float()).all())


# ---- towers ------------------------------------------------------------------------------------------------------------

def _model(arch, sd, max_batch):
    import clip_retrieval_b200 as m

    return m.B200Clip(arch, device=0, max_batch=max_batch).load_state_dict(sd)


def _check_tower(model, arch, sd, px, ids, what):
    import torch

    with torch.no_grad():
        ri = siglip_ref.image_features(sd, arch, px).double()
        rt = siglip_ref.text_features(sd, arch, ids).double()
    gi = model.encode_image(px.cuda()).cpu().double()
    gt = model.encode_text(ids.cuda()).cpu().double()
    for name, g, r in (("image", gi, ri), ("text", gt, rt)):
        d = cos_dist(g, r)
        rel = float(((g.norm(dim=-1) - r.norm(dim=-1)).abs() / r.norm(dim=-1)).max())
        assert d.max() <= COS_TOL and rel <= 0.02, "%s %s: 1 - cos %.2e, norm %.2e" % (what, name, d.max(), rel)
    return gi, gt


@pytest.mark.timeout(300)
def test_tiny_tower_matches_golden_and_oracle():
    gm = golden_module()
    arch = tiny_arch()
    sd = gm.state_dict()
    px, ids = gm.inputs()
    model = _model(arch, sd, 4)
    gi, gt = _check_tower(model, arch, sd, px, ids, "tiny")
    gold = np.load(os.path.join(GOLDEN, "siglip_tiny.npz"))
    assert cos_dist(gi, gold["image"]).max() <= COS_TOL and cos_dist(gt, gold["text"]).max() <= COS_TOL
    s = sensitise(sd)
    _check_tower(_model(arch, s, 4), arch, s, structured_images(4, arch.image_size, 2), captions(4, arch, 2),
                 "tiny sensitised")


def _table_cases():
    import clip_retrieval_b200 as m

    return sorted(m.SIGLIP_ARCHS)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("key", _table_cases())
def test_table_tower_two_layers(key):
    """Every table entry at its real widths, heads, image size and context, 2 layers per tower, sensitised weights and
    structured inputs (a smaller vocabulary: the embedding table's size does not change the arithmetic)."""
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import synthetic_state_dict

    a = m.SIGLIP_ARCHS[key]
    a = replace(a, vision=replace(a.vision, layers=2), text=replace(a.text, layers=2), vocab_size=1000)
    sd = sensitise(synthetic_state_dict(a, seed=1))
    model = _model(a, sd, 4)
    _check_tower(model, a, sd, structured_images(3, a.image_size, 1), captions(3, a, 1), key)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("key", ["open_clip:ViT-B-16-SigLIP", "open_clip:ViT-SO400M-14-SigLIP-384"])
def test_full_depth_tower(key):
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import synthetic_state_dict

    a = replace(m.SIGLIP_ARCHS[key], vocab_size=1000)
    sd = synthetic_state_dict(a, seed=2)
    _check_tower(_model(a, sd, 2), a, sd, structured_images(2, a.image_size, 3), captions(2, a, 3), key)


# ---- entry points -------------------------------------------------------------------------------------------------------

@pytest.mark.timeout(600)
def test_entry_points():
    """Batch-1 graph replay bit-identical to eager; chunk seams (max_batch 2, batch 5) and 40-sample batches (the
    128 x 256 GEMM) within the bar; host and device entries bit-identical."""
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import synthetic_state_dict

    a = m.SIGLIP_ARCHS["open_clip:ViT-SO400M-14-SigLIP"]
    a = replace(a, vision=replace(a.vision, layers=2), text=replace(a.text, layers=2), vocab_size=1000)
    sd = sensitise(synthetic_state_dict(a, seed=4))
    px, ids = structured_images(40, a.image_size, 4), captions(40, a, 4)
    model = _model(a, sd, 64)
    one = [model.embed_image_device(px[:1].cuda(), dtype=torch.float32).cpu() for _ in range(3)]
    onet = [model.embed_text_device(ids[:1].cuda(), dtype=torch.float32).cpu() for _ in range(3)]
    assert all(torch.equal(one[0], o) for o in one) and all(torch.equal(onet[0], o) for o in onet)
    _check_tower(model, a, sd, px, ids, "batch 40")
    dev_i = model.embed_image_device(px.cuda()).cpu().numpy()
    dev_t = model.embed_text_device(ids.cuda()).cpu().numpy()
    assert np.array_equal(model.embed_image(px), dev_i) and np.array_equal(model.embed_text(ids), dev_t)
    with pytest.raises(ValueError):
        model.embed_text(ids[:, :8].numpy())
    small = _model(a, sd, 2)
    _check_tower(small, a, sd, px[:5], ids[:5], "max_batch 2, batch 5")


@pytest.mark.timeout(900)
def test_so400m_384_load_clip_mapper_and_service(tmp_path):
    """A synthetic SO400M-384 checkpoint and the tiny tokenizer under a clip_cache_path; load_clip returns a 1152-d
    model, the SigLIP transform and a 64-token tokenizer; ClipMapper's image_rgb8 path (GPU squash, 0.5 / 0.5) equals
    the host transform's embeddings bit for bit, with a ragged last batch; one text query through B200KnnService."""
    import torch
    from PIL import Image

    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import synthetic_state_dict
    from clip_retrieval_b200.preprocess import to_rgb8
    from oracle import synth_ref

    name = "open_clip:ViT-SO400M-14-SigLIP-384/webli"
    arch = m.SIGLIP_ARCHS["open_clip:ViT-SO400M-14-SigLIP-384"]
    torch.save(synthetic_state_dict(arch, seed=6), str(tmp_path / "ViT-SO400M-14-SigLIP-384.bin"))
    (tmp_path / arch.tokenizer).mkdir(parents=True)
    tiny_tokenizer_json(str(tmp_path / arch.tokenizer / "tokenizer.json"))
    m.load_clip.cache_clear()
    model, preprocess, tokenizer = m.load_clip(clip_model=name, use_jit=False, warmup_batch_size=4,
                                               clip_cache_path=str(tmp_path))
    assert model.arch.embed_dim == 1152
    assert tokenizer(["a photo of a cat"]).shape == (1, 64)
    mapper = m.ClipMapper(True, True, False, False, name, False, "", warmup_batch_size=4, clip_cache_path=str(tmp_path))
    assert mapper.model is model
    folder = os.path.join(GOLDEN, "ref_images")
    ims = [Image.open(os.path.join(folder, f)) for f in sorted(os.listdir(folder))][:5]
    while len(ims) < 5:
        ims.append(ims[len(ims) % max(1, len(ims))].transpose(Image.FLIP_LEFT_RIGHT))
    host = torch.stack([preprocess(im) for im in ims])
    toks = tokenizer(["a photo of the cat", "red car", "x", "blue dog on the car", "photo"])
    rgb = [to_rgb8(im) for im in ims]
    full = mapper({"image_rgb8": rgb[:4], "text_tokens": toks[:4], "image_filename": list("abcd"), "text": list("abcd")})
    last = mapper({"image_rgb8": rgb[4:], "text_tokens": toks[4:], "image_filename": ["e"], "text": ["e"]})
    want = mapper({"image_tensor": host, "text_tokens": toks, "image_filename": list("abcde"), "text": list("abcde")})
    assert np.array_equal(full["image_embs"], want["image_embs"][:4])
    assert np.array_equal(last["image_embs"], want["image_embs"][4:])
    assert np.array_equal(full["text_embs"], want["text_embs"][:4])
    d, n, k = 1152, 3000, 20
    X = synth_ref.rows_f16(n, d, seed=5)
    idx = m.B200FlatIndex(d)
    idx.add(X)
    res = m.ClipResource(model, tokenizer=tokenizer, image_index=idx, text_index=idx)
    svc = m.B200KnnService({"siglip": res})
    got = svc.query(text_input="a photo of a cat", modality="image", num_images=k, num_result_ids=k, deduplicate=False)
    q = svc.compute_query_device(res, text_input="a photo of a cat")
    assert q.shape == (1, d) and abs(float(q.norm()) - 1.0) < 1e-3
    D, I = idx.search_device(q, k)
    assert [r["id"] for r in got] == [int(i) for i in I[0].cpu().numpy()]
    del svc, res, mapper, model
    m.load_clip.cache_clear()
    torch.cuda.empty_cache()
