"""open_clip's XLM-RoBERTa CLIPs on the GPU: the MLP head and the token-length kernel at kernel level, the tiny model
against the HuggingFace golden and the oracle, both real-size synthetic models (text against the fp32 oracle, images
bit for bit against the CLIP of the same image tower), padding invariance, the mapper and the query service."""
import os
import shutil

import numpy as np
import pytest

import mclip_ref
import xlmr_clip_ref
from test_xlmr_clip_cpu import open_clip_state_dict, tiny_arch

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3
U = 2.0 ** -24


def _gamma(n):
    return n * U / (1 - n * U)


def run_head(x, lengths, w1, w2, B, T):
    """b200_mean_mlp_head_device on CUDA x bf16 [B*T, w] with nn.Linear weights w1 [h, w], w2 [D, h] (fp32)."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    h, w = w1.shape
    D = w2.shape[0]
    w1T, w2T = w1.t().contiguous(), w2.t().contiguous()
    d_len = torch.as_tensor(lengths, dtype=torch.int32, device="cuda")
    hid = torch.full((B, h), float("nan"), device="cuda")
    feat = torch.full((B, D), float("nan"), device="cuda")
    out = torch.full((B, D), float("nan"), device="cuda")
    check(lib.b200_mean_mlp_head_device(x.data_ptr(), B, T, w, d_len.data_ptr(), w1T.data_ptr(), h, w2T.data_ptr(), D,
                                        hid.data_ptr(), feat.data_ptr(), out.data_ptr(), 0, 1, 0,
                                        torch.cuda.current_stream().cuda_stream), "mean_mlp_head")
    torch.cuda.synchronize()
    return hid, feat, out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("shape", [(768, 640, 512), (1024, 1024, 1024), (200, 72, 100)])
@pytest.mark.parametrize("B", [1, 3, 64, 1024])
def test_mlp_head_matches_float64(B, shape):
    """The head against float64 under a per-element bound (u = 2^-24, gamma(n) = n u / (1 - n u)):
      mean:    each column is an fp32 sum of L terms in order, then a division: |m^ - m| <= e_m = gamma(L) mean|x|;
      layer 1: a column is 4 quarters of two interleaved fma chains, added in a tree, so a product passes through at
               most w/8 + 4 roundings: e_1 = gamma(w/8 + 4) |W1| (|m| + e_m) + |W1| e_m;
      GELU:    |gelu'| <= 1.13, and 0.5 y (1 + erff(y / sqrt 2)) adds at most 8 u |y| (erff within 2 ulp):
               e_g = 1.13 e_1 + 8 u |y_1|;
      layer 2: e_2 = gamma(h/8 + 4) |W2| (|g| + e_g) + |W2| e_g.
    The normalised rows against the kernel's own features in float64: the sum of squares passes through at most
    D/256 + 14 roundings, then a square root and a division: |out - f / |f|| <= (gamma(D/256 + 14) + 3u) |f| / |f|."""
    import torch

    w, h, D = shape
    T = 5
    g = torch.Generator(device="cuda").manual_seed(B * 7 + w)
    x = torch.randn(B * T, w, device="cuda", generator=g).bfloat16()
    lengths = [(b * 3) % T + 1 for b in range(B)]
    w1 = torch.randn(h, w, device="cuda", generator=g) * w ** -0.5
    w2 = torch.randn(D, h, device="cuda", generator=g) * h ** -0.5
    hid, feat, out = run_head(x, lengths, w1, w2, B, T)
    xd = x.double().view(B, T, w)
    L = torch.as_tensor(lengths, device="cuda", dtype=torch.float64)
    live = (torch.arange(T, device="cuda")[None, :] < L[:, None]).double()
    m = (xd * live[:, :, None]).sum(1) / L[:, None]
    e_m = _gamma(T) * (xd.abs() * live[:, :, None]).sum(1) / L[:, None]
    W1, W2 = w1.double(), w2.double()
    y1 = m @ W1.t()
    e1 = _gamma(w / 8 + 4) * ((m.abs() + e_m) @ W1.abs().t()) + e_m @ W1.abs().t()
    gl = 0.5 * y1 * (1 + torch.erf(y1 / 2 ** 0.5))
    e_g = 1.13 * e1 + 8 * U * y1.abs()
    y2 = gl @ W2.t()
    e2 = _gamma(h / 8 + 4) * ((gl.abs() + e_g) @ W2.abs().t()) + e_g @ W2.abs().t()
    err = (feat.double() - y2).abs()
    assert bool((err <= e2 * (1 + 1e-9) + 1e-30).all()), "max err / bound %g" % float((err / e2).max())
    assert bool(((hid.double() - gl).abs() <= e_g * (1 + 1e-9) + 1e-30).all())
    f = feat.double()
    n = f.norm(dim=1, keepdim=True)
    bound = (_gamma(D / 256 + 14) + 3 * U) * f.abs() / n
    assert bool(((out.double() - f / n).abs() <= bound + 1e-30).all())


@pytest.mark.timeout(120)
def test_token_lengths_kernel():
    import torch
    from clip_retrieval_b200._lib import lib, check

    rng = np.random.default_rng(4)
    for B, T in ((1, 1), (7, 77), (300, 77), (5, 512)):
        ids = rng.integers(0, 9, size=(B, T)).astype(np.int64)
        ids[ids == 1] = 5
        cut = rng.integers(0, T + 1, size=B)
        cut[0], cut[-1] = T, (0 if B > 1 else T)   # one row without padding, one of padding only
        for b in range(B):
            ids[b, cut[b]:] = 1                   # right padding from cut[b]: none when cut[b] == T, all when 0
        if B > 2:
            ids[1, T // 2] = 1                    # a pad id inside a row: the first one counts
            ids[1, T // 2 + 1:] = 3
        want = np.where((ids == 1).any(1), (ids == 1).argmax(1), T)
        d_ids = torch.as_tensor(ids, device="cuda")
        d_len = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        check(lib.b200_text_lengths_device(d_ids.data_ptr(), B, T, 1, d_len.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream), "text_lengths")
        assert np.array_equal(d_len.cpu().numpy(), want), (B, T)
        assert want[0] == T and (B == 1 or want[-1] == 0)


@pytest.mark.timeout(300)
def test_tiny_model_matches_golden_and_oracle():
    import torch
    import clip_retrieval_b200 as m

    arch = tiny_arch()
    cfg, hidden = xlmr_clip_ref.CONFIGS["tiny"]
    sd_text = xlmr_clip_ref.make_state_dict(cfg, hidden, seed=0)
    model = m.B200XLMRClip(arch, device=0, max_batch=4).load_state_dict(open_clip_state_dict(arch, sd_text))
    z = np.load(os.path.join(GOLDEN, "xlmr_clip_tiny.npz"))
    ids = z["ids"]                                                   # 9 rows: three chunks of max_batch 4
    raw = model.encode_text(torch.as_tensor(ids).cuda())
    assert raw.dtype == torch.float32 and tuple(raw.shape) == (len(ids), cfg.out_dim)
    raw = raw.cpu().numpy()
    assert (1 - mclip_ref.cosine(raw, z["features"])).max() <= COS_TOL
    np.testing.assert_allclose(np.linalg.norm(raw, axis=1), np.linalg.norm(z["features"], axis=1), rtol=2e-2)
    emb = model.embed_text_device(ids, dtype=torch.float32).cpu().numpy()
    assert (1 - mclip_ref.cosine(emb, xlmr_clip_ref.embeddings(sd_text, cfg, ids))).max() <= COS_TOL
    np.testing.assert_allclose(np.linalg.norm(emb, axis=1), 1.0, atol=1e-5)
    # host entry: checked, trimmed to the longest row, and bit-identical to the device entry at T = 77
    host = model.embed_text(ids)
    assert host.dtype == np.float16 and np.array_equal(host, model.embed_text_device(ids).cpu().numpy())
    assert np.array_equal(model.embed_text(torch.as_tensor(ids[:3])), host[:3])
    bad = ids.copy()
    bad[1, 60] = 9
    with pytest.raises(ValueError, match="row 1"):
        model.embed_text(bad)
    with pytest.raises(m.B200Error):                                 # the image-only handle has no text tower
        model.visual.embed_text_device(torch.zeros(1, 77, dtype=torch.long, device="cuda"))
    img = torch.randn(2, 3, 32, 32, device="cuda")
    assert tuple(model.embed_image(img).shape) == (2, cfg.out_dim)


def _synth_ids(lengths, seed):
    cfg = xlmr_clip_ref.CONFIGS["tiny"][0]
    ids = mclip_ref.synth_ids(lengths, mclip_ref.EncCfg(**{**cfg.__dict__, "vocab_size": 250002}), seed=seed)
    out = np.full((len(lengths), 77), 1, dtype=np.int64)
    out[:, :ids.shape[1]] = ids
    return out


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name,clip", [("xlm-roberta-base-ViT-B-32", "open_clip:ViT-B-32"),
                                       ("xlm-roberta-large-ViT-H-14", "open_clip:ViT-H-14")])
def test_real_size_synthetic_model(name, clip):
    """load_clip of the synthetic real-size model.  Text at lengths 2..77 against the fp32 oracle (1 - cos <= 1e-3),
    and padding invariance: each caption alone (T = its length), in a batch of another order and at T = 77 gives the
    same bits, on the device and on the host entry.  Images: bit-identical to B200Clip of the CLIP with the same
    visual.* tensors."""
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import synthetic_state_dict
    from clip_retrieval_b200.xlmr_clip import split_state_dict, synthetic_state_dict as xlmr_sd

    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model, preprocess, _ = m.load_clip("synthetic:open_clip:" + name, warmup_batch_size=4)
    assert isinstance(model, m.B200XLMRClip) and model.arch.image_size == 224
    arch = model.arch
    cfg, _ = xlmr_clip_ref.CONFIGS[name]
    text_sd = split_state_dict(xlmr_sd(arch, seed=0), arch)[1]
    lengths = [2, 9, 33, 64, 77]
    ids = _synth_ids(lengths, seed=5)
    got = model.embed_text_device(ids, dtype=torch.float32).cpu().numpy()
    ref = xlmr_clip_ref.embeddings(text_sd, cfg, ids)
    worst = (1 - mclip_ref.cosine(got, ref)).max()
    print("%s 1-cos %.3e" % (name, worst))
    assert worst <= COS_TOL, worst
    del text_sd
    for b, L in enumerate(lengths):
        alone = model.embed_text_device(ids[b:b + 1, :L], dtype=torch.float32).cpu().numpy()
        assert np.array_equal(alone[0], got[b]), "%s: caption %d alone differs from the batch" % (name, b)
    order = [3, 0, 4, 2, 1]
    mixed = model.embed_text_device(ids[order], dtype=torch.float32).cpu().numpy()
    assert np.array_equal(mixed, got[order])
    assert np.array_equal(model.embed_text(ids), model.embed_text_device(ids).cpu().numpy())
    # images
    clip_model = m.B200Clip(m.ARCHS[clip], device=0, max_batch=4).load_state_dict(
        synthetic_state_dict(m.ARCHS[clip], seed=0))
    g = torch.Generator(device="cuda").manual_seed(2)
    img = torch.randn(3, 3, 224, 224, device="cuda", generator=g)
    assert torch.equal(model.encode_image(img), clip_model.encode_image(img))
    assert np.array_equal(model.embed_image(img.cpu()), clip_model.embed_image(img.cpu()))
    assert torch.equal(model.embed_image_device(img[:1]), clip_model.embed_image_device(img[:1]))


@pytest.mark.timeout(600)
def test_mapper_with_xlmr_clip():
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.xlmr_clip import XLMR_CLIP_ARCHS, split_state_dict, synthetic_state_dict
    from oracle import clip_ref

    name = "synthetic:open_clip:xlm-roberta-base-ViT-B-32"
    mapper = m.ClipMapper(True, True, True, False, name, True, "", warmup_batch_size=4)
    plain = m.ClipMapper(True, True, True, False, "synthetic:open_clip:ViT-B-32", True, "", warmup_batch_size=4)
    arch = XLMR_CLIP_ARCHS["xlm-roberta-base-ViT-B-32"]
    cfg, _ = xlmr_clip_ref.CONFIGS["xlm-roberta-base-ViT-B-32"]
    text_sd = split_state_dict(synthetic_state_dict(arch, seed=0), arch)[1]
    ccfg = clip_ref.CONFIGS["ViT-B/32"]
    for bs in (4, 3):                                                # a ragged last batch
        ids = _synth_ids([5, 40, 12, 77][:bs], seed=bs)
        item = {"image_tensor": clip_ref.synth_images(bs, ccfg, seed=bs), "text_tokens": torch.as_tensor(ids),
                "image_filename": ["f%d" % i for i in range(bs)], "text": ["t%d" % i for i in range(bs)],
                "metadata": ["{}"] * bs}
        out = mapper(item)
        for k in ("image_embs", "text_embs"):
            assert out[k].dtype == np.float16 and out[k].shape == (bs, 512)
        assert (1 - mclip_ref.cosine(out["text_embs"], xlmr_clip_ref.embeddings(text_sd, cfg, ids))).max() <= COS_TOL
        assert np.array_equal(out["image_embs"], plain(item)["image_embs"])
        assert out["text"] == item["text"] and out["image_filename"] == item["image_filename"]


@pytest.mark.timeout(600)
def test_service_and_micro_batcher(tmp_path):
    """query(text_input=...) through a tokenizer folder returns the ids of a search with the oracle's query (ids
    whose oracle scores lie closer than the query difference allows may swap); MicroBatcher results equal
    one-at-a-time searches bit for bit."""
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.xlmr_clip import XLMR_CLIP_ARCHS, XLMRTokenizer, split_state_dict, synthetic_state_dict

    os.makedirs(tmp_path / "xlm-roberta-base")
    shutil.copy(os.path.join(GOLDEN, "mclip_unigram_tokenizer.json"), tmp_path / "xlm-roberta-base" / "tokenizer.json")
    model, _, tok = m.load_clip("synthetic:open_clip:xlm-roberta-base-ViT-B-32/laion5b_s13b_b90k",
                                warmup_batch_size=1, clip_cache_path=str(tmp_path))
    assert isinstance(tok, XLMRTokenizer)
    arch = XLMR_CLIP_ARCHS["xlm-roberta-base-ViT-B-32"]
    cfg, _ = xlmr_clip_ref.CONFIGS["xlm-roberta-base-ViT-B-32"]
    text_sd = split_state_dict(synthetic_state_dict(arch, seed=0), arch)[1]
    n, d, k = 5000, 512, 20
    rng = np.random.default_rng(9)
    X = rng.standard_normal((n, d)).astype(np.float32)
    X = (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float16)
    idx = m.B200FlatIndex(d, device=0)
    idx.add(X)
    res = m.ClipResource(model=model, tokenizer=tok, device="cuda", image_index=idx)
    svc = m.B200KnnService({"idx": res})
    for text in ("ein Hund", "un chat sur le tapis", "  a   cat on the mat "):
        q = svc.compute_query_device(res, text_input=text).cpu().numpy()[0]
        q_ref = xlmr_clip_ref.embeddings(text_sd, cfg, tok([text]).numpy())[0].astype(np.float64)
        assert 1 - mclip_ref.cosine(q, q_ref) <= COS_TOL
        out = svc.query(text_input=text, num_images=k, num_result_ids=k, deduplicate=False)
        ids = np.array([r["id"] for r in out])
        scores = X.astype(np.float64) @ q_ref
        kth = np.sort(scores)[::-1][k - 1]
        tol = 2 * np.linalg.norm(q - q_ref) + 1e-6
        assert len(set(ids.tolist())) == k and scores[ids].min() >= kth - tol
        assert set(np.nonzero(scores > kth + tol)[0].tolist()) <= set(ids.tolist())
        via_tokens = svc.query(text_tokens=tok([text]), num_images=k, num_result_ids=k, deduplicate=False)
        assert via_tokens == out
    rows = tok(["ein Hund", "le chat", "the mat", "x", "", "un chat sur le tapis"])
    mb = m.MicroBatcher(model, idx, max_batch=4, max_wait_ms=50, k=k)
    try:
        futs = [mb.submit(r) for r in rows]
        got = [f.result(timeout=120) for f in futs]
    finally:
        mb.close()
    assert mb.batches < len(rows)
    for r, (D, I) in zip(rows, got):
        D1, I1 = idx.search_device(model.embed_text_device(r[None].cuda(), dtype=torch.float32), k)
        assert np.array_equal(D, D1.cpu().numpy()[0]) and np.array_equal(I, I1.cpu().numpy()[0])
