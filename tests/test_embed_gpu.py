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
    """The fixed-epsilon LayerNorm entry under the float64 bound of test_embed_kernels_gpu.check_layernorm, at a few
    tower widths (every row class, in place included)."""
    from test_embed_kernels_gpu import check_layernorm

    for rows, w in ((1, 64), (77, 512), (1000, 768), (515, 1024), (33, 1280)):
        check_layernorm(w, rows, ((1e-5, None),))


def attention_ref64(qkv, B, T, heads, hd, causal):
    """float64 softmax(Q K^T hd^-0.5 [+ causal mask]) V of the bf16 qkv buffer, its per-element error bound, and P.

    Bound: |out - ref| <= 2^-8 |ref| + (2^-8 + 2 ds + 2^-18) * sum_t P_t |v_t|.
    - 2^-8 |ref|: the bf16 store.
    - 2^-8 * sum_t P_t |v_t|: both kernels round P to bf16 (relative 2^-8) before P.V, and normalise by the fp32 sum
      of the unrounded P.
    - ds: the fp32 error of a score, (hd / 16 + 2) * 2^-22 * max_t |q| . |k_t| * hd^-0.5 (see test_gemm_gpu.py); a
      score off by ds moves P_t by at most a factor exp(2 ds).
    - 2^-18: exp2f, the fp32 P.V sums and the final division.
    A key dropped or wrongly admitted moves the output by P_t |v_t|, which this bound only sees when P_t is large:
    the one-hot probes below check every key of the tile edges exactly."""
    import torch

    q, k, v = qkv.double().view(B, T, 3, heads, hd).permute(2, 0, 3, 1, 4)
    sc = hd ** -0.5
    s = (q @ k.transpose(-1, -2)) * sc
    mag = (q.abs() @ k.abs().transpose(-1, -2)) * sc
    if causal:
        mask = torch.ones(T, T, dtype=torch.bool, device=qkv.device).triu_(1)
        s = s.masked_fill(mask, float("-inf"))
        mag = mag.masked_fill(mask, 0.0)
    P = torch.softmax(s, -1)
    ds = (hd // 16 + 2) * 2.0 ** -22 * mag.amax(-1, keepdim=True)
    ref = P @ v
    spread = P @ v.abs()
    bound = 2.0 ** -8 * ref.abs() + (2.0 ** -8 + 2 * ds + 2.0 ** -18) * spread
    flat = lambda t: t.transpose(1, 2).reshape(B * T, heads * hd)   # noqa: E731
    return flat(ref), flat(bound), P


def run_attention(qkv, B, T, heads, w, causal):
    import torch
    from clip_retrieval_b200._lib import lib, check

    out = torch.full((B * T, w), float("nan"), device="cuda", dtype=torch.bfloat16)
    check(lib.b200_attention_bf16_device(qkv.data_ptr(), out.data_ptr(), B, T, heads, w, causal, 0,
                                         torch.cuda.current_stream().cuda_stream), "attention")
    torch.cuda.synchronize()
    return out


def assert_attention_close(out, ref, bound, what=""):
    import torch

    got = out.double()
    assert not torch.isnan(got).any(), what
    err = (got - ref).abs()
    assert bool((err <= bound).all()), "%s: max err / bound %g (max err %g)" % (what, (err / bound).max().item(),
                                                                                 err.max().item())


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,T,heads,hd,causal", [
    (2, 50, 12, 64, 0), (3, 77, 8, 64, 1), (2, 257, 16, 64, 0), (1, 257, 16, 80, 0), (2, 1, 2, 64, 0),
    (1, 77, 16, 64, 1), (1, 17, 2, 128, 1), (2, 33, 3, 96, 0),
])
def test_attention_matches_fp32_reference(B, T, heads, hd, causal):
    import torch

    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T + w)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal)
    ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
    assert_attention_close(out, ref, bound)


def _attention_shapes():
    """(T, heads, head dim, causal) of both towers of every architecture the model table names, and head dim 64 on
    both sides of the wgmma (T <= 320) / mma.sync switch and around the 64-row / 64-key blocks."""
    import clip_retrieval_b200 as m

    shapes = set()
    for a in m.ARCHS.values():
        shapes.add(((a.image_size // a.patch) ** 2 + 1, a.vision.heads, a.vision.width // a.vision.heads, 0))
        shapes.add((a.context_length, a.text.heads, a.text.width // a.text.heads, 1))
    for T in (63, 64, 65, 127, 128, 129, 319, 320, 321):
        for causal in (0, 1):
            shapes.add((T, 2, 64, causal))
    return sorted(shapes)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("T,heads,hd,causal", _attention_shapes())
def test_attention_model_shapes_match_float64(T, heads, hd, causal):
    """Every model's attention shape at B = 2 (T = 577 of ViT-L/14@336px, head dim 80 of ViT-H/14, its text tower)
    and the kernel switch-over, against the float64 reference."""
    import torch

    B, w = 2, heads * hd
    g = torch.Generator(device="cuda").manual_seed(T * 3 + w + causal)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal)
    ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
    assert_attention_close(out, ref, bound, "T=%d heads=%d hd=%d causal=%d" % (T, heads, hd, causal))


PROBE_DIMS = (0, 7, 8, 63)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T,hd", [(65, 64), (129, 64), (257, 64), (320, 64), (321, 64), (577, 64), (257, 80),
                                  (77, 64), (130, 128)])
def test_attention_one_hot_v_probes(T, hd, causal):
    """V is zero except one 1.0 per (sample, head): key t, dim j.  The output of that (sample, head) in dim j is then
    P[r, t] alone, and every other output is exactly 0.0: the rows a causal mask hides (r < t), every other dim
    (this pins the V-transpose swizzle), and the dims of the neighbouring samples' probes (a key of the next sample
    read through the same tile, or a row of another sample, would show there).  One launch of 5 samples x 9 heads
    carries each key of {0, 1, 31, 32, 63, 64, 65, T-2, T-1} (those < T) with 5 dims {0, 7, 8, 63, hd-1}; within a
    head, the 5 samples use 5 different dims."""
    import torch

    keys = sorted({t for t in (0, 1, 31, 32, 63, 64, 65, T - 2, T - 1) if t < T})
    dims = sorted(set(PROBE_DIMS + (hd - 1,)) | ({33} if hd - 1 in PROBE_DIMS else set()))
    B, heads = 5, len(keys)
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
    # P rounded to bf16, then the output: two roundings of at most 2^-8 each, plus the fp32 normalisation
    assert bool((err <= (2.0 ** -7 + 2.0 ** -12) * want[~zero]).all()), \
        "probe P[r, t]: max rel err %g" % (err / want[~zero]).max().item()
    if causal:
        for (b, h), (t, j) in probe.items():
            assert bool((out[b, :t, h, j] == 0).all()) and bool((out[b, t:, h, j] > 0).all()), (b, h, t, j)


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
    """Head dimension 64 on the wgmma attention kernel (T <= 320) at sequence lengths around its 64-row query tiles
    and 64-key blocks (T = 1, 128, 129, 256..260, 320) and at the ViT-L/14 batch shape, against the float64
    reference of the same bf16 inputs."""
    import torch

    hd = 64
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T + w)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal)
    ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
    assert_attention_close(out, ref, bound)


@pytest.mark.timeout(120)
def test_tcgen05_attention_second_key_block_dominates():
    """Scores whose maximum sits far into the row (keys >= 128 scaled up): the online softmax must rescale what it
    accumulated under the running maximum of the earlier key blocks."""
    import torch

    B, T, heads, hd = 3, 257, 4, 64
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(7)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    kview = qkv.view(B, T, 3, heads, hd)
    kview[0, 128:, 1] *= 6.0          # sample 0: every row sees much larger scores in the second block
    kview[1, 200:230, 1, 0] *= 6.0    # sample 1, head 0 only
    qkv = qkv.bfloat16()
    out = run_attention(qkv, B, T, heads, w, 0)
    ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, 0)
    assert_attention_close(out, ref, bound)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,T,heads,causal", [(3, 257, 4, 0), (2, 77, 3, 1), (2, 200, 2, 1), (1, 264, 2, 0), (2, 16, 2, 0)])
def test_tcgen05_attention_variants_are_bit_identical(B, T, heads, causal):
    """Work decomposition changes loads and scheduling, not arithmetic: a sample's attention output must not depend on
    the batch it runs in or on repeated launches (one (query tile, head, sample) per CTA; keys of the next sample
    that a tile reads are masked).  Every sample alone, twice, must reproduce the batched result bit for bit."""
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
    """Inputs that break a softmax built on a precomputed score bound; the kernels run an online softmax with the
    running row maximum.  (a) Keys with a huge norm that are nearly orthogonal to every query.  (b) Large aligned
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
