"""Parity of the CUDA embed path (through the C ABI / the ClipMapper drop-in) against the CPU oracle
and the HuggingFace-generated golden vectors.  Floating point: north_star's bound is 1e-3 cosine
(1 - cos <= 1e-3) between embeddings; the path computes in bf16 with fp32 accumulation/statistics.
Component kernels are compared with plain fp32 PyTorch references of the same op."""
import os

import numpy as np
import pytest

from oracle import clip_ref

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3


def _arch(m, cfg):
    return m.ClipArch(cfg.embed_dim, cfg.image_size, cfg.patch,
                      m.Tower(cfg.vision.width, cfg.vision.layers, cfg.vision.heads, cfg.vision.mlp),
                      m.Tower(cfg.text.width, cfg.text.layers, cfg.text.heads, cfg.text.mlp),
                      cfg.context_length, cfg.vocab_size, cfg.quick_gelu)


def _model(name, max_batch):
    import clip_retrieval_b200 as m

    cfg = clip_ref.CONFIGS[name]
    sd = clip_ref.make_state_dict(cfg, seed=0)
    model = m.B200Clip(_arch(m, cfg), device=0, max_batch=max_batch)
    model.load_state_dict(sd)
    return model, cfg, sd


@pytest.mark.timeout(120)
def test_layernorm_matches_fp32_reference():
    import torch
    from clip_retrieval_b200._lib import lib, check

    for rows, w in ((1, 64), (77, 512), (1000, 768), (515, 1024), (33, 1280)):
        g = torch.Generator(device="cuda").manual_seed(rows + w)
        x = (torch.randn(rows, w, device="cuda", generator=g) * 3 + 0.5).bfloat16()
        ga = torch.randn(w, device="cuda", generator=g)
        be = torch.randn(w, device="cuda", generator=g)
        out = torch.empty_like(x)
        check(lib.b200_layernorm_bf16_device(x.data_ptr(), out.data_ptr(), ga.data_ptr(), be.data_ptr(), rows, w, 0,
                                             torch.cuda.current_stream().cuda_stream), "ln")
        ref = torch.nn.functional.layer_norm(x.float(), (w,), ga, be, 1e-5)
        err = (out.float() - ref).abs()
        assert bool((err <= ref.abs() * 2 ** -7 + 1e-2).all()), "rows=%d w=%d max err %g" % (rows, w, err.max().item())


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,T,heads,hd,causal", [
    (2, 50, 12, 64, 0), (3, 77, 8, 64, 1), (2, 257, 16, 64, 0), (1, 257, 16, 80, 0), (2, 1, 2, 64, 0),
    (1, 77, 16, 64, 1), (1, 17, 2, 128, 1), (2, 33, 3, 96, 0),
])
def test_attention_matches_fp32_reference(B, T, heads, hd, causal):
    import torch
    from clip_retrieval_b200._lib import lib, check

    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T + w)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    out = torch.full((B * T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    check(lib.b200_attention_bf16_device(qkv.data_ptr(), out.data_ptr(), B, T, heads, w, causal, 0,
                                         torch.cuda.current_stream().cuda_stream), "attention")
    q, k, v = qkv.float().view(B, T, 3, heads, hd).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if causal:
        s = s + torch.full((T, T), float("-inf"), device="cuda").triu_(1)
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * T, w)
    err = (out.float() - ref).abs()
    assert not torch.isnan(out.float()).any()
    # P is rounded to bf16 before P.V and the output to bf16: 2^-7 relative + 2e-2 absolute
    assert bool((err <= ref.abs() * 2 ** -7 + 2e-2).all()), "max err %g" % err.max().item()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name,n,max_batch", [("tiny", 5, 2), ("tiny-gelu", 5, 8), ("ViT-B/32", 4, 4)])
def test_embeddings_match_oracle_and_hf_golden(name, n, max_batch):
    import torch

    model, cfg, sd = _model(name, max_batch)
    px = clip_ref.synth_images(n, cfg, seed=0)
    tk = clip_ref.synth_tokens(n, cfg, seed=0)
    gold = np.load(os.path.join(GOLDEN, "clip_%s.npz" % name.replace("/", "-")))
    # raw features (what model.encode_image returns) vs HF golden and oracle
    fi = model.encode_image(px.cuda()).cpu().numpy()
    ft = model.encode_text(tk.cuda()).cpu().numpy()
    assert fi.shape == (n, cfg.embed_dim) and fi.dtype == np.float32
    for got, ref_hf, ref_or in ((fi, gold["image_features"], clip_ref.encode_image(sd, cfg, px).numpy()),
                                (ft, gold["text_features"], clip_ref.encode_text(sd, cfg, tk).numpy())):
        assert (1 - clip_ref.cosine(got, ref_hf)).max() <= COS_TOL
        assert (1 - clip_ref.cosine(got, ref_or)).max() <= COS_TOL
        # magnitudes too (cosine ignores scale): within 2% of the fp32 norm
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), np.linalg.norm(ref_or, axis=1), rtol=2e-2)
    # the mapper call: normalised fp16 numpy, host buffers in
    ei = model.embed_image(px)
    et = model.embed_text(tk)
    assert ei.dtype == np.float16 and et.dtype == np.float16 and ei.shape == (n, cfg.embed_dim)
    assert (1 - clip_ref.cosine(ei, clip_ref.mapper_image(sd, cfg, px))).max() <= COS_TOL
    assert (1 - clip_ref.cosine(et, clip_ref.mapper_text(sd, cfg, tk))).max() <= COS_TOL
    np.testing.assert_allclose(np.linalg.norm(ei.astype(np.float32), axis=1), 1.0, atol=2e-3)
    # device path == host path bit for bit (same kernels, only the copies differ)
    assert np.array_equal(model.embed_image_device(px.cuda()).cpu().numpy(), ei)


@pytest.mark.timeout(600)
def test_vit_l14_matches_oracle():
    import torch

    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model, cfg, sd = _model("ViT-L/14", 2)
    px = clip_ref.synth_images(2, cfg, seed=1)
    tk = clip_ref.synth_tokens(2, cfg, seed=1)
    ei, et = model.embed_image(px), model.embed_text(tk)
    ci = 1 - clip_ref.cosine(ei, clip_ref.mapper_image(sd, cfg, px))
    ct = 1 - clip_ref.cosine(et, clip_ref.mapper_text(sd, cfg, tk))
    assert ci.max() <= COS_TOL and ct.max() <= COS_TOL, (ci, ct)


@pytest.mark.timeout(300)
def test_mapper_drop_in_contract():
    """The reference's own mapper test pins shape[0] and dtype float16 (tests/test_clip_inference/
    test_mapper.py:37-38); the runner/writer read exactly these five keys (runner.py:44-47,
    writer.py:43-56)."""
    import torch
    import clip_retrieval_b200 as m

    mapper = m.ClipMapper(enable_image=True, enable_text=True, enable_metadata=True, use_mclip=False,
                          clip_model="synthetic:ViT-B/32", use_jit=True, mclip_model="", warmup_batch_size=4)
    cfg = clip_ref.CONFIGS["ViT-B/32"]
    for bs in (4, 3, 1):  # short last batches
        item = {
            "image_tensor": clip_ref.synth_images(bs, cfg, seed=bs),
            "text_tokens": clip_ref.synth_tokens(bs, cfg, seed=bs),
            "image_filename": ["f%d" % i for i in range(bs)],
            "text": ["t%d" % i for i in range(bs)],
            "metadata": ["{}"] * bs,
        }
        out = mapper(item)
        assert set(out) == {"image_embs", "text_embs", "image_filename", "text", "metadata"}
        assert out["image_embs"].shape[0] == bs and out["image_embs"].dtype == np.float16
        assert out["text_embs"].shape == (bs, 512) and out["text_embs"].dtype == np.float16
        assert out["image_filename"] == item["image_filename"] and out["text"] == item["text"]
    off = m.ClipMapper(False, False, False, False, "synthetic:ViT-B/32", True, "", warmup_batch_size=4)
    res = off({"image_tensor": None})
    assert res["image_embs"] is None and res["text_embs"] is None and res["metadata"] is None
    with pytest.raises(NotImplementedError):
        m.ClipMapper(True, True, False, True, "synthetic:ViT-B/32", True, "x")


@pytest.mark.timeout(300)
def test_zero_feature_row_is_nan_like_reference():
    """`features /= features.norm()` has no epsilon (mapper.py:58): an all-zero feature row must not
    be silently 'fixed'.  Built by zeroing the output projection."""
    import torch

    model, cfg, sd = _model("tiny", 2)
    sd = dict(sd)
    sd["visual.proj"] = torch.zeros_like(sd["visual.proj"])
    model.load_state_dict(sd)
    out = model.embed_image(clip_ref.synth_images(2, cfg))
    assert np.isnan(out.astype(np.float32)).all()


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,T,heads,causal", [(2, 257, 16, 0), (3, 77, 8, 1), (2, 50, 12, 0), (1, 1, 2, 0), (5, 128, 4, 1),
                                              (1, 320, 2, 0), (40, 257, 16, 0), (3, 260, 2, 0), (2, 256, 2, 1), (7, 129, 3, 0), (2, 258, 3, 1)])
def test_tcgen05_attention_matches_fp32_reference(B, T, heads, causal):
    """The shapes that pinned the Blackwell tensor-core attention, now on the attention kernel the model runs on H100:
    head dimension 64 at sequence lengths around its 16-row query blocks and 32-key blocks (T = 1, 128, 129, 256..260,
    320) and at the ViT-L/14 batch shape, against a plain fp32 PyTorch softmax(QK^T)V of the same bf16 inputs."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    hd = 64
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T + w)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    out = torch.full((B * T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    check(lib.b200_attention_bf16_device(qkv.data_ptr(), out.data_ptr(), B, T, heads, w, causal, 0,
                                         torch.cuda.current_stream().cuda_stream), "attention")
    q, k, vv = qkv.float().view(B, T, 3, heads, hd).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if causal:
        s = s + torch.full((T, T), float("-inf"), device="cuda").triu_(1)
    ref = (torch.softmax(s, -1) @ vv).transpose(1, 2).reshape(B * T, w)
    err = (out.float() - ref).abs()
    assert not torch.isnan(out.float()).any()
    assert bool((err <= ref.abs() * 2 ** -7 + 2e-2).all()), "max err %g" % err.max().item()


@pytest.mark.timeout(120)
def test_tcgen05_attention_second_key_block_dominates():
    """Scores whose maximum sits far into the row (keys >= 128 scaled up): a guard for any softmax
    variant that processes the key columns in blocks with a running reference maximum."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    B, T, heads, hd = 3, 257, 4, 64
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(7)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    kview = qkv.view(B, T, 3, heads, hd)
    kview[0, 128:, 1] *= 6.0          # sample 0: every row sees much larger scores in the second block
    kview[1, 200:230, 1, 0] *= 6.0    # sample 1, head 0 only
    qkv = qkv.bfloat16()
    out = torch.full((B * T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    q, k, vv = qkv.float().view(B, T, 3, heads, hd).permute(2, 0, 3, 1, 4)
    ref = (torch.softmax((q @ k.transpose(-1, -2)) * hd ** -0.5, -1) @ vv).transpose(1, 2).reshape(B * T, w)
    check(lib.b200_attention_bf16_device(qkv.data_ptr(), out.data_ptr(), B, T, heads, w, 0, 0,
                                         torch.cuda.current_stream().cuda_stream), "attention")
    err = (out.float() - ref).abs()
    assert not torch.isnan(out.float()).any()
    assert bool((err <= ref.abs() * 2 ** -7 + 2e-2).all()), "max err %g" % err.max().item()


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,T,heads,causal", [(3, 257, 4, 0), (2, 77, 3, 1), (2, 200, 2, 1), (1, 264, 2, 0), (2, 16, 2, 0)])
def test_tcgen05_attention_variants_are_bit_identical(B, T, heads, causal):
    """Work decomposition changes loads and scheduling, not arithmetic: a sample's attention output must not depend on
    the batch it runs in or on repeated launches (one (head, sample) per block; the query-block split per warp
    depends on T only).  Every sample alone, twice, must reproduce the batched result bit for bit."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    w = heads * 64
    g = torch.Generator(device="cuda").manual_seed(T * 7 + heads)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    st = torch.cuda.current_stream().cuda_stream
    full = torch.full((B * T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    check(lib.b200_attention_bf16_device(qkv.data_ptr(), full.data_ptr(), B, T, heads, w, causal, 0, st), "attention")
    torch.cuda.synchronize()
    assert not torch.isnan(full.float()).any()
    for b in range(B):
        for _ in range(2):
            one = torch.full((T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
            src = qkv[b * T:(b + 1) * T].contiguous()
            check(lib.b200_attention_bf16_device(src.data_ptr(), one.data_ptr(), 1, T, heads, w, causal, 0, st), "attention")
            torch.cuda.synchronize()
            assert torch.equal(one, full[b * T:(b + 1) * T]), "sample %d differs from its batched result" % b


@pytest.mark.timeout(120)
@pytest.mark.parametrize("T,causal", [(257, 0), (77, 1), (200, 0)])
def test_tcgen05_attention_single_pass_bound_and_fallback(T, causal):
    """Inputs that broke a bound-based softmax, on the attention kernel the model runs on H100 (online softmax with the
    running row maximum).  (a) Keys with a huge norm that are nearly orthogonal to every query.  (b) Large aligned
    scores (spread over > 100 log2 units) must neither overflow nor lose the small terms that still matter.  (c) A
    sample whose neighbour in the batch holds non-finite activations must not be contaminated."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    B, heads, hd = 3, 4, 64
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(T)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = qkv.view(B, T, 3, heads, hd)
    # (a) sample 0: key 3 of every head is 400x larger but lives (almost) in one coordinate the queries avoid
    view[0, :, 0, :, 0] = 0.0
    view[0, 3, 1] = 0.0
    view[0, 3, 1, :, 0] = 4000.0
    # (b) sample 1: queries and a few keys strongly aligned and large
    view[1, :, 0, 0] *= 6.0
    view[1, 10:14, 1, 0] = view[1, 20, 0, 0] * 1.5
    qkv = qkv.bfloat16()
    ref_in = qkv.clone()
    # (c) sample 2 is poisoned AFTER the reference is computed for samples 0/1 on clean data
    poisoned = qkv.clone()
    poisoned.view(B, T, 3, heads, hd)[2] = float("inf")
    out = torch.full((B * T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    check(lib.b200_attention_bf16_device(poisoned.data_ptr(), out.data_ptr(), B, T, heads, w, causal, 0,
                                         torch.cuda.current_stream().cuda_stream), "attention")
    q, k, vv = ref_in.float().view(B, T, 3, heads, hd).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if causal:
        s = s + torch.full((T, T), float("-inf"), device="cuda").triu_(1)
    ref = (torch.softmax(s, -1) @ vv).transpose(1, 2).reshape(B, T, w)
    got = out.float().view(B, T, w)
    for b in (0, 1):
        assert not torch.isnan(got[b]).any() and not torch.isinf(got[b]).any(), "sample %d" % b
        err = (got[b] - ref[b]).abs()
        assert bool((err <= ref[b].abs() * 2 ** -6 + 3e-2).all()), "sample %d max err %g" % (b, err.max().item())
