"""The ResNet CLIP image tower on the GPU (csrc/conv.cu, csrc/resnet.cu): the implicit 3x3 convolution against a float64
conv2d of the same bf16 operands, one-hot tap probes, the ReLU epilogue on the 128- and 256-wide GEMMs, the stem
gather / pool / token kernels, the towers against oracle/resnet_ref.py and the torch.nn golden, and the drop-in paths
(load_clip, ClipMapper, B200KnnService).

Convolution bound, per element: the GEMM bound of test_gemm_gpu.py with K = 9 * C64 and S = conv2d(|x|, |w|); ReLU
has slope <= 1 and adds no rounding of its own.
"""
import math
import os

import numpy as np
import pytest

from oracle import clip_ref, resnet_ref

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3


def pack3x3(w):
    """[N, C, 3, 3] -> [N, 9 * C64] with column (3 r + s) * C64 + c (include/b200clip.h b200_conv_bf16_device)."""
    import torch

    N, C = w.shape[:2]
    c64 = (C + 63) // 64 * 64
    out = torch.zeros(N, 9, c64, dtype=w.dtype, device=w.device)
    out[:, :, :C] = w.permute(0, 2, 3, 1).reshape(N, 9, C)
    return out.reshape(N, 9 * c64).contiguous()


def conv(x, w, ksize, bias=None, residual=None, act=0, bn=0, check=True):
    """b200_conv_bf16_device on NHWC x [B, H, W, C] -> [B*H*W, N] bf16."""
    import torch
    from clip_retrieval_b200._lib import lib, GemmEpilogueC, check as chk

    B, H, W, C = x.shape
    N = w.shape[0]
    out = torch.empty(B * H * W, N, dtype=torch.bfloat16, device="cuda")
    p = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    ep = GemmEpilogueC(p(bias), p(residual), 0, 0, 0, 0, 0, act)
    wp = pack3x3(w) if ksize == 3 else w.reshape(N, C).contiguous()
    rc = lib.b200_conv_bf16_device(x.data_ptr(), B, H, W, C, wp.data_ptr(), N, ksize, out.data_ptr(), ep, bn, 0,
                                   torch.cuda.current_stream().cuda_stream)
    if check:
        chk(rc, "conv")
    torch.cuda.synchronize()
    return out if check else rc


def conv_ref64(x, w, ksize, bias, residual, act):
    """(y, bound): float64 conv2d of the bf16 operands, + bias, + residual, relu; the bound of the module docstring."""
    import torch
    import torch.nn.functional as F

    B, H, W, C = x.shape
    N = w.shape[0]
    xd = x.permute(0, 3, 1, 2).double()
    pre = F.conv2d(xd, w.double(), padding=ksize // 2)
    S = F.conv2d(xd.abs(), w.double().abs(), padding=ksize // 2)
    pre = pre.permute(0, 2, 3, 1).reshape(-1, N)
    S = S.permute(0, 2, 3, 1).reshape(-1, N)
    K = (9 * ((C + 63) // 64 * 64)) if ksize == 3 else C
    e = (math.ceil(K / 16) + 2) * 2.0 ** -22 * S
    if bias is not None:
        pre = pre + bias.double()
    e = e + 2.0 ** -22 * pre.abs()
    y = pre
    if residual is not None:
        y = y + residual.double()
        e = e + 2.0 ** -22 * residual.double().abs()
    if act == 3:
        y = y.clamp_min(0)
    return y, 2.0 ** -8 * (y.abs() + e) + e


def _operands(B, H, W, C, N, seed, k=3):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, C, k, k, device="cuda", generator=g) * (2.0 / (C * k * k)) ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g) * 0.5
    r = torch.randn(B * H * W, N, device="cuda", generator=g).bfloat16()
    return x, w, b, r


def _check(out, y, bound, what):
    from test_gemm_gpu import assert_close

    assert_close(out, y, bound, what)


def model_conv_shapes():
    """Every distinct (H, Cin, Cout) of the implicit convolutions of the five models."""
    import clip_retrieval_b200 as m

    out = set()
    for k in ("RN50", "RN101", "RN50x4", "RN50x16", "RN50x64"):
        a = m.RESNET_ARCHS[k]
        w = a.width
        out.add((a.image_size // 2, w // 2, w // 2))
        out.add((a.image_size // 2, w // 2, w))
        for s, H in enumerate((a.image_size // 4, a.image_size // 4, a.image_size // 8, a.image_size // 16)):
            # block 0 of stages 1..3 runs conv2 before its pool (at the stage's input size), the others after it
            out.add((H, w << s, w << s))
            if s > 0:
                out.add((H // 2, w << s, w << s))
    return sorted(out)


# ---- the implicit convolution -------------------------------------------------------------------------------------

@pytest.mark.timeout(900)
@pytest.mark.parametrize("H,C,N", model_conv_shapes())
def test_conv_model_shapes(H, C, N):
    """Every implicit convolution the five models run, bias + ReLU (the tower's epilogue), one image."""
    x, w, b, _ = _operands(1, H, H, C, N, seed=H * 7 + C)
    out = conv(x, w, 3, bias=b, act=3)
    y, bound = conv_ref64(x, w, 3, b, None, 3)
    _check(out, y, bound, "conv H=%d C=%d N=%d" % (H, C, N))


CASES = [
    # (B, H, W, C, N): channel tails, tiny and odd spatial sizes, B*H*W not a multiple of 128
    (3, 9, 9, 8, 64), (2, 7, 7, 40, 80), (1, 9, 9, 48, 96), (2, 12, 12, 80, 80), (1, 18, 18, 96, 128),
    (2, 9, 9, 160, 160), (5, 1, 1, 64, 64), (3, 2, 2, 128, 256), (4, 7, 7, 512, 512), (3, 7, 9, 64, 72),
    (2, 33, 31, 64, 64), (1, 56, 56, 64, 64),
]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("B,H,W,C,N", CASES)
@pytest.mark.parametrize("epi", ["none", "bias_relu", "bias_res_relu"])
@pytest.mark.parametrize("bn", [128, 64, 32])
def test_conv_epilogues_and_tails(B, H, W, C, N, epi, bn):
    x, w, b, r = _operands(B, H, W, C, N, seed=B + H + C + N)
    bias = b if epi != "none" else None
    res = r if epi == "bias_res_relu" else None
    act = 0 if epi == "none" else 3
    out = conv(x, w, 3, bias=bias, residual=res, act=act, bn=bn)
    y, bound = conv_ref64(x, w, 3, bias, res, act)
    _check(out, y, bound, "conv %s bn=%d" % ((B, H, W, C, N), bn))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("B,H,W,C", [(2, 5, 7, 8), (1, 9, 9, 40), (2, 4, 4, 96), (1, 3, 3, 160)])
def test_tap_probes_reproduce_the_shifted_input_exactly(B, H, W, C):
    """Output channel j of a one-hot weight at (channel c_j, tap r_j, s_j) is the input channel c_j shifted by
    (r_j - 1, s_j - 1), bit for bit, with exact zeros outside the image."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(C)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).bfloat16()
    taps = [(c, r, s) for r in range(3) for s in range(3) for c in sorted({0, C // 2, C - 1})]
    N = (len(taps) + 7) // 8 * 8
    w = torch.zeros(N, C, 3, 3, device="cuda", dtype=torch.bfloat16)
    for j, (c, r, s) in enumerate(taps):
        w[j, c, r, s] = 1.0
    out = conv(x, w, 3).view(B, H, W, N)
    xp = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)   # [B, H+2, W+2, C]
    for j, (c, r, s) in enumerate(taps):
        want = xp[:, r:r + H, s:s + W, c]
        assert torch.equal(out[..., j], want), (c, r, s)
    assert not bool(out[..., len(taps):].any())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("res", [False, True])
def test_relu_epilogue_on_both_gemm_widths(bn, res):
    """The 1x1 convolution (the GEMM of the NHWC rows) with bias + ReLU and bias + residual + ReLU on the 128-wide
    and the persistent 256-wide kernel: inside the bound, and the two widths bit-identical."""
    import torch

    B, H, C, N = 4, 28, 256, 512   # 3136 rows x 512: 50 tiles of 128 x 256
    x, w, b, r = _operands(B, H, H, C, N, seed=11, k=1)
    resid = r if res else None
    out = conv(x, w, 1, bias=b, residual=resid, act=3, bn=bn)
    y, bound = conv_ref64(x, w, 1, b, resid, 3)
    _check(out, y, bound, "1x1 relu bn=%d" % bn)
    other = conv(x, w, 1, bias=b, residual=resid, act=3, bn=384 - bn)
    assert torch.equal(out, other)
    assert float(out.float().min()) >= 0.0


def test_public_gemm_entries_still_refuse_relu():
    """ACT_RELU is internal: b200_gemm_bf16_device and the epilogue entry keep accepting 0..2 only."""
    import torch
    from test_gemm_gpu import gemm, operands

    A, W, b, R = operands(128, 64, 64, 1)
    out = torch.empty(128, 64, dtype=torch.bfloat16, device="cuda")
    assert gemm(A, W, out, bias=b, act=3) != 0
    x, w, _, _ = _operands(1, 4, 4, 8, 8, seed=1)
    assert conv(x, w, 3, act=1, check=False) != 0   # the 3x3 convolution takes none or relu only


# ---- small kernels ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,S", [(2, 64), (1, 224), (3, 30)])
def test_stem_gather_is_exact(B, S):
    import torch
    import torch.nn.functional as F
    from clip_retrieval_b200._lib import lib, check

    g = S // 2
    px = torch.randn(B, 3, S, S, device="cuda")
    cols = torch.full((B * g * g, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    check(lib.b200_stem_gather_device(px.data_ptr(), B, S, cols.data_ptr(), 0, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    ref = F.unfold(px, 3, padding=1, stride=2).transpose(1, 2).reshape(B * g * g, 27).bfloat16()
    assert torch.equal(cols[:, :27], ref)
    assert bool(torch.isnan(cols[:, 27:].float()).all())


@pytest.mark.parametrize("B,H,C,k", [(2, 16, 64, 2), (3, 7, 256, 2), (1, 112, 128, 2), (2, 9, 40, 3)])
def test_avgpool_matches_float64(B, H, C, k):
    import torch
    import torch.nn.functional as F
    from clip_retrieval_b200._lib import lib, check

    x = torch.randn(B, H, H, C, device="cuda").bfloat16()
    Ho = H // k
    out = torch.empty(B, Ho, Ho, C, dtype=torch.bfloat16, device="cuda")
    check(lib.b200_avgpool_bf16_device(x.data_ptr(), B, H, H, C, k, out.data_ptr(), 0,
                                       torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    y = F.avg_pool2d(x.permute(0, 3, 1, 2).double(), k).permute(0, 2, 3, 1)
    e = (k * k) * 2.0 ** -23 * F.avg_pool2d(x.permute(0, 3, 1, 2).double().abs(), k).permute(0, 2, 3, 1)
    _check(out, y, 2.0 ** -8 * (y.abs() + e) + e, "avgpool")


@pytest.mark.parametrize("B,HW,C", [(2, 4, 512), (3, 49, 2048), (1, 196, 4096)])
def test_attnpool_tokens_match_float64(B, HW, C):
    import torch
    from clip_retrieval_b200._lib import lib, check

    x = torch.randn(B * HW, C, device="cuda").bfloat16()
    pos = torch.randn(HW + 1, C, device="cuda") * 0.1
    out = torch.empty(B * (HW + 1), C, dtype=torch.bfloat16, device="cuda")
    check(lib.b200_attnpool_tokens_device(x.data_ptr(), B, HW, C, pos.data_ptr(), out.data_ptr(), 0,
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    xd = x.double().view(B, HW, C)
    y = torch.cat([xd.mean(1, keepdim=True), xd], 1) + pos.double()
    e = torch.cat([(HW + 2) * 2.0 ** -23 * xd.abs().mean(1, keepdim=True), torch.zeros_like(xd)], 1)
    e = e + 2.0 ** -23 * (y.abs() + pos.double().abs())
    _check(out.view(B, HW + 1, C), y, 2.0 ** -8 * (y.abs() + e) + e, "attnpool tokens")


# ---- towers ------------------------------------------------------------------------------------------------------------

def _oracle_image(sd, arch, px):
    """oracle/resnet_ref.py in fp32 on the GPU, TF32 off for convolutions and matmuls."""
    import torch

    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        sd_dev = {k: v.cuda() for k, v in sd.items() if k.startswith("visual.")}
        return resnet_ref.encode_image(sd_dev, arch, px.cuda()).cpu().numpy()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
        torch.cuda.empty_cache()


def _images_apart(ref_i, what):
    """The oracle's features of the first two images differ by 1 - cos >= IMAGES_APART: the inputs can fail the bar."""
    from test_resnet_cpu import IMAGES_APART

    d = 1 - clip_ref.cosine(ref_i[0], ref_i[1])
    print("\n%s: images 1 - cos %.3g" % (what, d))
    assert d >= IMAGES_APART, (what, d)


def _check_tower(arch, sd, px, seed, what, discriminating=True):
    """encode_image / encode_text of px and seeded captions against the fp32 oracles: 1 - cos <= 1e-3, norms within
    2 %; the host entry stores the device entry's bits; with `discriminating`, the images are told apart (above)."""
    import clip_retrieval_b200 as m

    n = px.shape[0]
    model = m.B200Clip(arch, device=0, max_batch=n).load_state_dict(sd)
    tk = clip_ref.synth_tokens(n, arch, seed=seed)
    fi = model.encode_image(px.cuda()).cpu().numpy()
    ft = model.encode_text(tk.cuda()).cpu().numpy()
    ei = model.embed_image(px)
    assert np.array_equal(model.embed_image_device(px.cuda()).cpu().numpy(), ei)
    del model
    ref_i = _oracle_image(sd, arch, px)
    ref_t = resnet_ref.encode_text(sd, arch, tk).numpy()
    if discriminating:
        _images_apart(ref_i, what)
    for kind, got, ref in (("image", fi, ref_i), ("text", ft, ref_t)):
        d = 1 - clip_ref.cosine(got, ref)
        print("\n%s %s: 1 - cos max %.3g" % (what, kind, d.max()))
        assert d.max() <= COS_TOL, (what, kind, d)
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), np.linalg.norm(ref, axis=1), rtol=2e-2)
    n_ref = ref_i / np.linalg.norm(ref_i, axis=1, keepdims=True)
    assert (1 - clip_ref.cosine(ei, n_ref)).max() <= COS_TOL
    return fi


def _check_case(case):
    """A tower case of test_resnet_cpu.tower_cases on its weights and structured images: the inputs on which
    test_resnet_cpu.py shows every named wrong forward outside the bar and a bf16 stand-in inside half of it."""
    from test_resnet_cpu import tower_cases, tower_inputs

    a, sd, px = tower_inputs(case)
    _check_tower(a, sd, px, tower_cases()[case][1], case)


@pytest.mark.timeout(600)
def test_tiny_on_structured_images():
    _check_case("tiny")


@pytest.mark.timeout(600)
def test_tiny_matches_golden_and_oracle():
    """The golden's own inputs (plain weights, noise images): pins the forward against torch.nn, not a bar that can
    fail on its own (the test above is that)."""
    import importlib.util

    import clip_retrieval_b200 as m

    spec = importlib.util.spec_from_file_location("make_rn_golden", os.path.join(GOLDEN, "make_rn_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    sd = m.synthetic_state_dict(gen.TINY, seed=0)
    fi = _check_tower(gen.TINY, sd, clip_ref.synth_images(gen.N, gen.TINY, seed=0), 0, "tiny golden",
                      discriminating=False)
    gold = np.load(os.path.join(GOLDEN, "clip_tiny-rn.npz"))["image"]
    assert (1 - clip_ref.cosine(fi, gold)).max() <= COS_TOL


@pytest.mark.timeout(900)
@pytest.mark.parametrize("key", ["RN50", "RN101", "RN50x4", "RN50x16", "RN50x64"])
def test_one_block_per_stage_at_real_widths(key):
    """Real widths, image size and attention-pool heads (T = 50 / 50 / 82 / 145 / 197), one block per stage."""
    _check_case(key + "-1block")


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("key", ["RN50", "RN50x4"])
def test_full_depth_matches_oracle(key):
    _check_case(key + "-full")


@pytest.mark.timeout(600)
def test_batch1_graph_replay_is_bit_identical_to_eager():
    """Batch 1 runs eagerly, is captured, then replayed: every call stores the same bits; so does a handle with graphs
    off."""
    import torch

    import clip_retrieval_b200 as m

    a = m.RESNET_ARCHS["RN50"]
    sd = m.synthetic_state_dict(a, seed=3)
    model = m.B200Clip(a, device=0, max_batch=4).load_state_dict(sd)
    px = clip_ref.synth_images(1, a, seed=5).cuda()
    outs = [model.encode_image(px) for _ in range(4)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    assert torch.isfinite(outs[0]).all()
    del model
    prev = os.environ.get("B200_GRAPHS")
    os.environ["B200_GRAPHS"] = "0"   # read when the handle is created
    try:
        eager = m.B200Clip(a, device=0, max_batch=4).load_state_dict(sd)
    finally:
        if prev is None:
            del os.environ["B200_GRAPHS"]
        else:
            os.environ["B200_GRAPHS"] = prev
    for _ in range(3):
        assert torch.equal(eager.encode_image(px), outs[0])


# ---- drop-ins ----------------------------------------------------------------------------------------------------------

@pytest.mark.timeout(900)
def test_load_clip_synthetic_and_state_dict_file(tmp_path):
    """load_clip of `synthetic:RN50x4` (288 px transform) and of an RN50 state_dict saved in OpenAI's key layout, with
    num_batches_tracked and the scalar entries of the TorchScript archives, and the BPE tokenizer.  The images are
    structured (test_resnet_cpu.structured_images), on which a full-depth tower tells them apart, so the oracle check
    can fail."""
    import shutil

    import torch
    from torchvision import transforms as T

    import clip_retrieval_b200 as m

    model, pre, tok = m.load_clip("synthetic:RN50x4", warmup_batch_size=2, clip_cache_path=None)
    assert isinstance(model.arch, m.ResNetArch) and model.arch.image_size == 288
    sizes = [t.size for t in pre.transforms if isinstance(t, (T.Resize, T.CenterCrop))]
    assert sizes[0] == 288 and tuple(sizes[1]) == (288, 288)

    from test_resnet_cpu import structured_images

    a = m.RESNET_ARCHS["RN50"]
    sd = m.synthetic_state_dict(a, seed=4)
    assert sd["visual.bn1.num_batches_tracked"].dtype == torch.int64
    sd.update({"input_resolution": torch.tensor(224), "context_length": torch.tensor(77),
               "vocab_size": torch.tensor(49408), "logit_scale": torch.tensor(4.6052)})
    torch.save(sd, str(tmp_path / "RN50.pt"))
    shutil.copy(os.path.join(GOLDEN, "bpe_tiny.txt.gz"), str(tmp_path / "bpe_simple_vocab_16e6.txt.gz"))
    model, pre, tok = m.load_clip("RN50", warmup_batch_size=2, clip_cache_path=str(tmp_path))
    assert model.arch == a
    toks = tok(["a photo of a cat", "a dog"])
    assert toks.shape == (2, 77) and int(toks[0, 0]) == tok.encoder["<|startoftext|>"]
    px = structured_images(2, a.image_size, seed=6)
    got = model.encode_image(px.cuda()).cpu().numpy()
    ref = _oracle_image(sd, a, px)
    _images_apart(ref, "RN50.pt")
    d = 1 - clip_ref.cosine(got, ref)
    print("\nRN50.pt image: 1 - cos max %.3g" % d.max())
    assert d.max() <= COS_TOL
    t = model.embed_text(toks)
    assert t.shape == (2, 1024) and np.isfinite(t.astype(np.float32)).all()
    m.load_clip.cache_clear()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["synthetic:RN50x16", "synthetic:open_clip:RN50x64/openai"])
def test_mapper_image_tensor_and_rgb8(name):
    import torch

    import clip_retrieval_b200 as m

    mapper = m.ClipMapper(True, True, False, False, name, False, "", warmup_batch_size=3)
    a = mapper.model.arch
    n_px = a.image_size
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((n_px + 40, n_px + 13), (200, 640), (n_px, n_px))]
    tens = m.B200Preprocess(n_px)(imgs).cpu()
    tk = clip_ref.synth_tokens(3, a, seed=2)
    out = mapper({"image_tensor": tens, "text_tokens": tk, "image_filename": list("abc"), "text": list("abc")})
    assert out["image_embs"].shape == (3, a.embed_dim) and out["text_embs"].shape == (3, a.embed_dim)
    np.testing.assert_allclose(np.linalg.norm(out["image_embs"].astype(np.float32), axis=1), 1.0, atol=2e-3)
    via_rgb8 = mapper({"image_rgb8": imgs, "text_tokens": tk, "image_filename": list("abc"), "text": list("abc")})
    via_rgb8 = via_rgb8["image_embs"]
    assert np.array_equal(via_rgb8, out["image_embs"])
    del mapper
    m.load_clip.cache_clear()
    torch.cuda.empty_cache()


@pytest.mark.timeout(600)
def test_knn_service_query_on_rn50():
    import torch

    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import SimpleTokenizer
    from oracle import synth_ref

    model, _, _ = m.load_clip("synthetic:RN50", warmup_batch_size=1, clip_cache_path=None)
    d, n, k = model.arch.embed_dim, 3000, 20
    X = synth_ref.rows_f16(n, d, seed=5)
    idx = m.B200FlatIndex(d)
    idx.add(X)
    tok = SimpleTokenizer(os.path.join(GOLDEN, "bpe_tiny.txt.gz"))
    res = m.ClipResource(model, tokenizer=tok, image_index=idx, text_index=idx)
    svc = m.B200KnnService({"rn50": res})
    got = svc.query(text_input="a photo of a cat", modality="image", num_images=k, num_result_ids=k, deduplicate=False)
    q = svc.compute_query_device(res, text_input="a photo of a cat")
    assert q.shape == (1, d) and abs(float(q.norm()) - 1.0) < 1e-3
    D, I = idx.search_device(q, k)
    assert [r["id"] for r in got] == [int(i) for i in I[0].cpu().numpy()]
    del svc, res, model
    m.load_clip.cache_clear()
    torch.cuda.empty_cache()
