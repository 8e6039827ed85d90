"""The multilingual text towers on the GPU (use_mclip): key-length attention and the encoder embedding at kernel level
(LayerNorm with an epsilon and the linear head are in test_embed_kernels_gpu.py); the whole encoder against the
HuggingFace goldens and the fp32 oracle, at the real XLM-R-Large and DistilBERT-multilingual sizes too; padding invariance; the mapper and the query service.
Ids come from the goldens or are synthetic: no test here needs the `tokenizers` package."""
import os
from dataclasses import replace

import numpy as np
import pytest

import mclip_ref
from test_embed_gpu import assert_attention_close, attention_ref64

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3


def _arch(cfg):
    import clip_retrieval_b200 as m

    return m.EncoderArch(cfg.family, cfg.layers, cfg.width, cfg.heads, cfg.ffn, cfg.vocab_size, cfg.max_positions,
                         cfg.type_vocab_size, cfg.pad_token_id, cfg.eps, cfg.out_dim, cfg.proj_bias)


def _encoder(cfg, sd, max_batch=8, max_tokens=None):
    import clip_retrieval_b200 as m

    return m.B200TextEncoder(_arch(cfg), device=0, max_batch=max_batch, max_tokens=max_tokens).load_state_dict(sd)


def run_attention_len(qkv, lengths, B, T, heads, w):
    import torch
    from clip_retrieval_b200._lib import lib, check

    d_len = torch.as_tensor(lengths, dtype=torch.int32, device="cuda")
    out = torch.full((B * T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    check(lib.b200_attention_len_bf16_device(qkv.data_ptr(), d_len.data_ptr(), out.data_ptr(), B, T, heads, w, 0,
                                             torch.cuda.current_stream().cuda_stream), "attention_len")
    torch.cuda.synchronize()
    return out


def _lengths(T):
    return sorted({T, 1, max(1, T // 2), max(1, T - 1), max(1, (3 * T) // 4), min(T, 17)})


@pytest.mark.timeout(300)
@pytest.mark.parametrize("T", [1, 17, 64, 65, 128, 320, 321, 512])
def test_key_length_attention_matches_float64(T):
    """Sample b against the float64 attention of its own first len[b] tokens; its rows >= len[b] are exactly 0.
    With every len[b] = T the result is the kernel without lengths, bit for bit."""
    import torch
    from test_embed_gpu import run_attention

    heads, hd = 2, 64
    w = heads * hd
    lengths = _lengths(T)
    B = len(lengths)
    g = torch.Generator(device="cuda").manual_seed(7 * T)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    out = run_attention_len(qkv, lengths, B, T, heads, w).view(B, T, w)
    for b, L in enumerate(lengths):
        src = qkv.view(B, T, 3 * w)[b, :L].contiguous()
        ref, bound, _ = attention_ref64(src, 1, L, heads, hd, 0)
        assert_attention_close(out[b, :L], ref, bound, "T=%d len=%d" % (T, L))
        assert bool((out[b, L:] == 0).all()), "T=%d len=%d: rows past the length are not zero" % (T, L)
    full = run_attention_len(qkv, [T] * B, B, T, heads, w)
    assert torch.equal(full, run_attention(qkv, B, T, heads, w, 0))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("T", [17, 64, 65, 129, 320, 321, 512])
def test_key_length_one_hot_v_probes(T):
    """V is zero except one 1.0 per (sample, head).  Head 0 carries it on a masked key (len <= t < T): every output
    of the sample is exactly 0.0.  Head 1 carries it on the last live key len - 1: its dim is P[r, len - 1] on the
    rows < len and 0.0 elsewhere, every other dim is 0.0."""
    import torch

    heads, hd = 2, 64
    w = heads * hd
    lengths = [L for L in _lengths(T) if L < T] or [max(1, T - 1)]
    B = len(lengths)
    g = torch.Generator(device="cuda").manual_seed(T + 11)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = qkv.view(B, T, 3, heads, hd)
    view[:, :, 2] = 0.0
    for b, L in enumerate(lengths):
        view[b, L + (T - 1 - L) * (b % 2), 2, 0, (7 * b) % hd] = 1.0       # a masked key: the first or the last
        view[b, L - 1, 2, 1, (5 * b + 3) % hd] = 1.0
    qkv = qkv.bfloat16()
    out = run_attention_len(qkv, lengths, B, T, heads, w).view(B, T, heads, hd).double()
    for b, L in enumerate(lengths):
        assert bool((out[b, :, 0] == 0).all()), "T=%d len=%d: a masked key contributes" % (T, L)
        j = (5 * b + 3) % hd
        rest = out[b, :, 1].clone()
        rest[:L, j] = 0
        assert bool((rest == 0).all()), (T, L)
        _, _, P = attention_ref64(qkv.view(B, T, 3 * w)[b, :L].contiguous(), 1, L, heads, hd, 0)
        want = P[0, 1, :, L - 1]
        err = (out[b, :L, 1, j] - want).abs()
        assert bool((err <= (2.0 ** -7 + 2.0 ** -12) * want).all()), (T, L, float((err / want).max()))


@pytest.mark.timeout(120)
@pytest.mark.parametrize("eps", [1e-12, 1e-5])
def test_layernorm_eps_matches_float64(eps):
    """The LayerNorm entry with an epsilon under the float64 bound of test_embed_kernels_gpu.check_layernorm, at the
    encoder widths; its rows include variances comparable to either epsilon."""
    from test_embed_kernels_gpu import check_layernorm

    for rows, w in ((1, 64), (77, 768), (515, 1024)):
        check_layernorm(w, rows, ((eps, eps),))


@pytest.mark.timeout(120)
@pytest.mark.parametrize("name", ["tiny-xlmr", "tiny-distilbert"])
def test_encoder_embedding_matches_fp32_sums(name):
    import torch
    from clip_retrieval_b200._lib import lib, check

    cfg = mclip_ref.CONFIGS[name]
    sd = {k: v.cuda() for k, v in mclip_ref.make_state_dict(cfg, seed=3).items()}
    B, T, w = 3, 21, cfg.width
    ids = torch.as_tensor(mclip_ref.synth_ids([21, 4, 9], cfg, seed=3)).cuda()
    ids[0, 5] = cfg.vocab_size + 7                   # out of range: clamped to the last row
    word = sd["embeddings.word_embeddings.weight"].bfloat16()
    tt = sd["embeddings.token_type_embeddings.weight"][0].contiguous() if cfg.type_vocab_size else None
    pos = sd["embeddings.position_embeddings.weight"]
    off = 2 if cfg.family == "xlm-roberta" else 0
    out = torch.empty(B * T, w, device="cuda", dtype=torch.bfloat16)
    check(lib.b200_encoder_embed_bf16_device(ids.data_ptr(), word.data_ptr(), tt.data_ptr() if tt is not None else None,
                                             pos.data_ptr(), off, sd["embeddings.LayerNorm.weight"].data_ptr(),
                                             sd["embeddings.LayerNorm.bias"].data_ptr(), cfg.eps, out.data_ptr(), B, T,
                                             w, cfg.vocab_size, 0, torch.cuda.current_stream().cuda_stream), "embed")
    torch.cuda.synchronize()
    x = word.float()[ids.clamp(0, cfg.vocab_size - 1)]
    if tt is not None:
        x = x + tt
    x = x + pos[off + torch.arange(T, device="cuda")]
    ref = torch.nn.functional.layer_norm(x, (w,), sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"],
                                         cfg.eps).view(B * T, w)
    err = (out.float() - ref).abs()
    assert bool((err <= ref.abs() * 2 ** -8 + 1e-5).all()), err.max().item()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", ["tiny-xlmr", "tiny-distilbert"])
def test_tiny_encoders_match_golden_and_oracle(name):
    import torch

    cfg = mclip_ref.CONFIGS[name]
    sd = mclip_ref.make_state_dict(cfg, seed=0)
    z = np.load(os.path.join(GOLDEN, "mclip_%s.npz" % name))
    enc = _encoder(cfg, sd, max_batch=4)          # 6 samples: two chunks
    raw = enc.embed_text_device(z["ids"], z["lengths"], normalize=False).cpu().numpy()
    assert (1 - mclip_ref.cosine(raw, z["features"])).max() <= COS_TOL
    np.testing.assert_allclose(np.linalg.norm(raw, axis=1), np.linalg.norm(z["features"], axis=1), rtol=2e-2)
    emb = enc.embed_text_device(z["ids"], z["lengths"])
    assert emb.dtype == torch.float32 and emb.shape == (len(z["lengths"]), cfg.out_dim)
    ref = mclip_ref.embeddings(sd, cfg, z["ids"], z["lengths"])
    assert (1 - mclip_ref.cosine(emb.cpu().numpy(), ref)).max() <= COS_TOL
    np.testing.assert_allclose(np.linalg.norm(emb.cpu().numpy(), axis=1), 1.0, atol=1e-5)
    # the host entry runs the same kernels
    assert np.array_equal(enc.embed_text(z["ids"], z["lengths"]), emb.cpu().numpy())
    f16 = enc.embed_text_device(z["ids"], z["lengths"], dtype=torch.float16)
    assert torch.equal(f16, emb.half())


@pytest.mark.timeout(300)
def test_concurrent_host_and_device_encodes_share_one_handle_safely():
    """The query service encodes from Flask threads: host-entry calls (legacy stream) and device-entry calls on a
    torch stream, from two threads on one handle, must each return what they return alone."""
    import threading

    import torch

    cfg = mclip_ref.CONFIGS["tiny-xlmr"]
    sd = mclip_ref.make_state_dict(cfg, seed=0)
    z = np.load(os.path.join(GOLDEN, "mclip_tiny-xlmr.npz"))
    ids, lengths = z["ids"], z["lengths"]
    enc = _encoder(cfg, sd, max_batch=8)
    want_host = enc.embed_text(ids, lengths)
    want_dev = enc.embed_text_device(ids, lengths, normalize=False).cpu().numpy()
    errs = []

    def host_worker():
        for _ in range(40):
            if not np.array_equal(enc.embed_text(ids, lengths), want_host):
                errs.append("host")

    def device_worker():
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for _ in range(40):
                out = enc.embed_text_device(ids, lengths, normalize=False)
                s.synchronize()
                if not np.array_equal(out.cpu().numpy(), want_dev):
                    errs.append("device")

    ts = [threading.Thread(target=host_worker), threading.Thread(target=device_worker)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs[:4]


def _padded(ids, pad, T):
    out = np.full((ids.shape[0], T), pad, dtype=np.int64)
    out[:, :ids.shape[1]] = ids
    return out


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["xlmr-large", "distilbert-multilingual"])
def test_real_size_synthetic_encoders(name):
    """Real-size seeded weights at lengths 2..128 (and 512 for XLM-R, on the mma.sync attention): 1 - cos <= 1e-3
    against the fp32 oracle.  Padding invariance: each sample alone (T = its length) and inside batches padded to
    T = 128 and 320 gives identical bits; padded to 321 (the other attention kernel) it stays within the bar."""
    import torch

    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cfg = mclip_ref.CONFIGS[name]
    sd = mclip_ref.make_state_dict(cfg, seed=5)
    lengths = [2, 17, 64, 65, 128]
    ids = mclip_ref.synth_ids(lengths, cfg, seed=5)
    enc = _encoder(cfg, sd, max_batch=len(lengths), max_tokens=512)
    got = enc.embed_text(ids, lengths)
    ref = mclip_ref.embeddings(sd, cfg, ids, lengths)
    worst = (1 - mclip_ref.cosine(got, ref)).max()
    print("%s 1-cos %.3e" % (name, worst))
    assert worst <= COS_TOL, worst
    for b, L in enumerate(lengths):
        alone = enc.embed_text(ids[b:b + 1, :L], [L])
        assert np.array_equal(alone[0], got[b]), "%s: sample %d alone differs from the batch" % (name, b)
    assert np.array_equal(enc.embed_text(_padded(ids, cfg.pad_token_id, 320), lengths), got)
    across = enc.embed_text(_padded(ids, cfg.pad_token_id, 321), lengths)
    assert (1 - mclip_ref.cosine(across, ref)).max() <= COS_TOL
    if cfg.family == "xlm-roberta":
        long_ids = mclip_ref.synth_ids([512], cfg, seed=6)
        g512 = enc.embed_text(long_ids, [512])
        r512 = mclip_ref.embeddings(sd, cfg, long_ids, [512])
        print("%s T=512 1-cos %.3e" % (name, (1 - mclip_ref.cosine(g512, r512)).max()))
        assert (1 - mclip_ref.cosine(g512, r512)).max() <= COS_TOL


@pytest.mark.timeout(120)
def test_zero_projection_gives_zero_rows():
    """normalized() divides a zero norm by 1: zero rows, never NaN (clip_back.py:194-197)."""
    import torch

    cfg = mclip_ref.CONFIGS["tiny-xlmr"]
    sd = mclip_ref.make_state_dict(cfg, seed=0)
    sd["projection.weight"] = torch.zeros_like(sd["projection.weight"])
    sd["projection.bias"] = torch.zeros_like(sd["projection.bias"])
    z = np.load(os.path.join(GOLDEN, "mclip_tiny-xlmr.npz"))
    out = _encoder(cfg, sd).embed_text(z["ids"], z["lengths"])
    assert np.array_equal(out, np.zeros_like(out))


class _GoldenTokenizer:
    """Stands in for the checkpoint tokenizer: the golden ids, one row per text."""

    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN, "mclip_%s.npz" % name))
        self.ids, self.lengths = z["ids"], z["lengths"]

    def __call__(self, texts):
        n = len(texts)
        L = self.lengths[:n]
        return self.ids[:n, :int(L.max())], L


@pytest.mark.timeout(300)
def test_mapper_use_mclip(tmp_path):
    import clip_retrieval_b200 as m
    from oracle import clip_ref
    from test_mclip_cpu import write_st_folder

    cfg = replace(mclip_ref.CONFIGS["tiny-distilbert"], out_dim=512)
    sd = mclip_ref.make_state_dict(cfg, seed=4)
    write_st_folder(str(tmp_path / "st"), sd, cfg)
    mapper = m.ClipMapper(True, True, True, True, "synthetic:ViT-B/32", True, str(tmp_path / "st"), warmup_batch_size=4)
    mapper.mclip.tokenizer = _GoldenTokenizer("tiny-distilbert")
    plain = m.ClipMapper(True, True, True, False, "synthetic:ViT-B/32", True, "", warmup_batch_size=4)
    ccfg = clip_ref.CONFIGS["ViT-B/32"]
    tok = mapper.mclip.tokenizer
    for bs in (4, 1):
        item = {"image_tensor": clip_ref.synth_images(bs, ccfg, seed=bs), "text_tokens": clip_ref.synth_tokens(bs, ccfg),
                "image_filename": ["f%d" % i for i in range(bs)], "text": ["t%d" % i for i in range(bs)],
                "metadata": ["{}"] * bs}
        out = mapper(item)
        assert out["text_embs"].dtype == np.float32 and out["text_embs"].shape == (bs, 512)
        ids, lengths = tok(item["text"])
        ref = mclip_ref.embeddings(sd, cfg, ids, lengths)
        assert (1 - mclip_ref.cosine(out["text_embs"], ref)).max() <= COS_TOL
        np.testing.assert_allclose(np.linalg.norm(out["text_embs"], axis=1), 1.0, atol=1e-5)
        assert np.array_equal(out["image_embs"], plain(item)["image_embs"])    # the image half is unchanged
        assert out["text"] == item["text"] and out["image_filename"] == item["image_filename"]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("aesthetic", [False, True])
def test_service_query_use_mclip(tmp_path, aesthetic):
    """query(use_mclip=True) over a flat index returns the ids of a search with the oracle's query; ids whose scores
    under the oracle query lie closer than the query difference can allow may swap (ties)."""
    import torch
    import clip_retrieval_b200 as m
    from test_mclip_cpu import write_mclip_folder

    cfg = mclip_ref.CONFIGS["tiny-xlmr"]
    sd = mclip_ref.make_state_dict(cfg, seed=0)
    write_mclip_folder(str(tmp_path / "mc"), sd, cfg)
    mm = m.load_mclip(str(tmp_path / "mc"))
    n, d, k = 5000, cfg.out_dim, 20
    rng = np.random.default_rng(8)
    X = rng.standard_normal((n, d)).astype(np.float32)
    X = (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float16)
    idx = m.B200FlatIndex(d, device=0)
    idx.add(X)
    aest = {9: rng.standard_normal(d).astype(np.float32)} if aesthetic else None
    res = m.ClipResource(model=None, device="cuda", image_index=idx, model_txt_mclip=mm, aesthetic_embeddings=aest)
    svc = m.B200KnnService({"idx": res})
    z = np.load(os.path.join(GOLDEN, "mclip_tiny-xlmr.npz"))
    for b in (1, 4):
        tokens = (z["ids"][b:b + 1, :z["lengths"][b]], z["lengths"][b:b + 1])
        kw = dict(aesthetic_score=9, aesthetic_weight=0.5) if aesthetic else {}
        q = svc.compute_query_device(res, use_mclip=True, mclip_tokens=tokens, **kw).cpu().numpy()[0]
        q_ref = mclip_ref.embeddings(sd, cfg, *tokens)[0].astype(np.float64)
        if aesthetic:
            q_ref = q_ref + aest[9] * 0.5
            q_ref = q_ref / np.linalg.norm(q_ref)
        assert 1 - mclip_ref.cosine(q, q_ref) <= COS_TOL
        out = svc.query(use_mclip=True, mclip_tokens=tokens, num_images=k, num_result_ids=k, deduplicate=False, **kw)
        ids = np.array([r["id"] for r in out])
        scores = X.astype(np.float64) @ q_ref
        kth = np.sort(scores)[::-1][k - 1]
        tol = 2 * np.linalg.norm(q - q_ref) + 1e-6
        assert len(set(ids.tolist())) == k and scores[ids].min() >= kth - tol
        assert set(np.nonzero(scores > kth + tol)[0].tolist()) <= set(ids.tolist())
    with pytest.raises(ValueError):
        m.B200KnnService({"x": m.ClipResource(model=None, device="cuda", image_index=idx)}).query(
            use_mclip=True, mclip_tokens=tokens)
    assert torch.cuda.is_available()
