"""The ConvNeXt CLIP image tower on the GPU (csrc/dwconv.cu, csrc/convnext.cu): dwconv7_ln, ln_s2d and the head
against float64, one-hot tap probes, the stem's patch GEMM with its zero K tail, the towers against
oracle/convnext_ref.py on the inputs of test_convnext_cpu.py (where every named wrong forward fails the bar and a bf16
stand-in uses 4 % of it), and the drop-in paths (load_clip, ClipMapper, B200KnnService).

Bounds, per element, with u = 2^-24 and the final bf16 rounding 2^-8 |y|:
- the convolution sum of 49 taps + bias in fp32: E = 50 u (conv2d(|x|, |w|) + |bias|);
- the LayerNorm on those sums: the error E moves (y - mean) by at most E + max E and rstd relatively by max E rstd, so
  the normalised value by |g| rstd (E + max E (1 + |n|)); its own fp32 statistics (C / 32 + 5 terms per sum) add
  2^-16 |g| (|n| + 1);
- a stored value within d of the exact one rounds to bf16 within 2^-8 (|y| + d) + d.
"""
import math
import os

import numpy as np
import pytest

from oracle import clip_ref, convnext_ref

pytestmark = pytest.mark.gpu

COS_TOL = 1e-3
U = 2.0 ** -24


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def dwconv(x, w49, bias, g=None, b=None, eps=1e-6):
    """b200_dwconv7_ln_bf16_device on NHWC x [B, H, W, C] -> [B, H, W, C] bf16."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    B, H, W, C = x.shape
    out = torch.empty_like(x)
    p = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    check(lib.b200_dwconv7_ln_bf16_device(x.data_ptr(), B, H, W, C, w49.data_ptr(), bias.data_ptr(), p(g), p(b), eps,
                                          out.data_ptr(), 0, _stream()), "dwconv7_ln")
    torch.cuda.synchronize()
    return out


def dwconv_ref64(x, w49, bias, g, b, eps):
    """(y, bound) of the module docstring, float64."""
    import torch
    import torch.nn.functional as F

    B, H, W, C = x.shape
    xd = x.permute(0, 3, 1, 2).double()
    wd = w49.double().t().reshape(C, 1, 7, 7)
    y = F.conv2d(xd, wd, bias.double(), padding=3, groups=C).permute(0, 2, 3, 1)
    S = F.conv2d(xd.abs(), wd.abs(), padding=3, groups=C).permute(0, 2, 3, 1)
    E = 50 * U * (S + bias.double().abs())
    if g is None:
        return y, 2.0 ** -8 * (y.abs() + E) + E
    mean = y.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((y - mean) ** 2).mean(-1, keepdim=True) + eps)
    n = (y - mean) * rstd
    gd = g.double().abs()
    Em = E.amax(-1, keepdim=True)
    d = gd * rstd * (E + Em * (1 + n.abs())) + 2.0 ** -16 * gd * (n.abs() + 1)
    out = n * g.double() + b.double()
    return out, 2.0 ** -8 * (out.abs() + d) + d


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    worst = float((err / bound).max())
    print("\n%s: max err / bound %.3g" % (what, worst))
    assert worst <= 1.0, what


def _dw_operands(B, H, C, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, H, C, generator=g).bfloat16().cuda()
    w49 = (torch.randn(49, C, generator=g) / 7).cuda()
    bias = (0.1 * torch.randn(C, generator=g)).cuda()
    gam = (1 + 0.2 * torch.randn(C, generator=g)).cuda()
    bet = (0.1 * torch.randn(C, generator=g)).cuda()
    return x, w49, bias, gam, bet


def model_dw_shapes():
    """Every (H, C) a table model's blocks run, and C = 3072 at H = 7, 8 and 80."""
    import clip_retrieval_b200 as m

    out = set()
    for a in m.CONVNEXT_ARCHS.values():
        for s in range(4):
            out.add((a.image_size // 4 >> s, a.dims[s]))
    out |= {(7, 3072), (8, 3072), (80, 3072)}
    return sorted(out)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("H,C", model_dw_shapes())
def test_dwconv7_ln_model_shapes(H, C):
    """Batch 1 and 3 (no multiple of any tile), with and without the LayerNorm, against float64."""
    for B in (1, 3):
        x, w49, bias, g, b = _dw_operands(B, H, C, seed=H * 10000 + C + B)
        eps = 1e-5 if C == 3072 else 1e-6
        y, bound = dwconv_ref64(x, w49, bias, g, b, eps)
        _check(dwconv(x, w49, bias, g, b, eps), y, bound, "dwconv7_ln B=%d H=%d C=%d" % (B, H, C))
        y, bound = dwconv_ref64(x, w49, bias, None, None, eps)
        _check(dwconv(x, w49, bias), y, bound, "dwconv7 B=%d H=%d C=%d (no LN)" % (B, H, C))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("B,H,W,C", [(2, 9, 11, 64), (1, 7, 7, 192), (1, 3, 20, 128)])
def test_tap_probes_reproduce_the_shifted_input_exactly(B, H, W, C):
    """With the LayerNorm off, weight 1 at one tap and bias 0: the output is the input shifted by (r - 3, s - 3), bit
    for bit, and exact zeros where the tap falls outside the map (all four borders)."""
    import torch

    x = torch.randn(B, H, W, C, generator=torch.Generator().manual_seed(H + W)).bfloat16().cuda()
    bias = torch.zeros(C, device="cuda")
    for k in range(49):
        r, s = divmod(k, 7)
        w49 = torch.zeros(49, C, device="cuda")
        w49[k] = 1.0
        got = dwconv(x, w49, bias)
        want = torch.zeros_like(x)
        dr, ds = r - 3, s - 3
        h0, h1 = max(0, -dr), min(H, H - dr)
        w0, w1 = max(0, -ds), min(W, W - ds)
        if h0 < h1 and w0 < w1:
            want[:, h0:h1, w0:w1] = x[:, h0 + dr:h1 + dr, w0 + ds:w1 + ds]
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (k, r, s)


def ln_s2d(x, g, b, eps):
    import torch
    from clip_retrieval_b200._lib import lib, check

    B, H, W, C = x.shape
    out = torch.empty(B * (H // 2) * (W // 2), 4 * C, dtype=torch.bfloat16, device="cuda")
    check(lib.b200_ln_s2d_bf16_device(x.data_ptr(), B, H, W, C, g.data_ptr(), b.data_ptr(), eps, out.data_ptr(), 0,
                                      _stream()), "ln_s2d")
    torch.cuda.synchronize()
    return out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("B,H,C", [(1, 56, 128), (3, 40, 256), (2, 16, 768), (1, 20, 1536), (3, 32, 384), (2, 4, 1536)])
def test_ln_s2d_places_columns_and_normalises(B, H, C):
    """Each pixel's LayerNorm lands at row (b, h / 2, w / 2), columns ((h & 1) 2 + (w & 1)) C + c: the index-coded
    check puts pixel (h, w)'s own offset into its row, so a misplaced row is off by O(1); the values against float64
    under the LayerNorm bound of the module docstring (the input is exact, E = 0)."""
    import torch
    import torch.nn.functional as F

    gen = torch.Generator().manual_seed(B * H + C)
    x = torch.randn(B, H, H, C, generator=gen)
    x = x + torch.arange(H * H, dtype=torch.float32).view(1, H, H, 1) * torch.linspace(-1, 1, C) * 0.05
    x = x.bfloat16().cuda()
    g = (1 + 0.2 * torch.randn(C, generator=gen)).cuda()
    b = (0.1 * torch.randn(C, generator=gen)).cuda()
    got = ln_s2d(x, g, b, 1e-6)
    xd = x.double()
    ref = F.layer_norm(xd, (C,), g.double(), b.double(), 1e-6)
    n = F.layer_norm(xd, (C,), None, None, 1e-6)
    d = 2.0 ** -16 * g.double().abs() * (n.abs() + 1)
    bound = 2.0 ** -8 * (ref.abs() + d) + d
    Ho = H // 2

    def s2d(t):
        return t.view(B, Ho, 2, Ho, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * Ho * Ho, 4 * C)

    _check(got, s2d(ref), s2d(bound), "ln_s2d B=%d H=%d C=%d" % (B, H, C))


def head(x, HW, g, b, eps, w1T, b1, w2T, D, normalize):
    import torch
    from clip_retrieval_b200._lib import lib, check

    B = x.shape[0] // HW
    C = x.shape[1]
    h = w1T.shape[1] if w1T is not None else 0
    pooled = torch.empty(B, C, device="cuda")
    hid = torch.empty(B, max(h, 1), device="cuda")
    feat = torch.empty(B, D, device="cuda")
    out = torch.empty(B, D, device="cuda")
    p = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    check(lib.b200_convnext_head_device(x.data_ptr(), B, HW, C, g.data_ptr(), b.data_ptr(), eps, p(w1T), p(b1), h,
                                        w2T.data_ptr(), D, pooled.data_ptr(), hid.data_ptr(), feat.data_ptr(),
                                        out.data_ptr(), 0, normalize, 0, _stream()), "convnext_head")
    torch.cuda.synchronize()
    return pooled, feat, out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("mlp", [False, True])
@pytest.mark.parametrize("B,HW,C,D", [(1, 49, 1024, 512), (3, 64, 1536, 768), (2, 100, 3072, 1024), (5, 4, 256, 64)])
def test_head_matches_float64(mlp, B, HW, C, D):
    """Mean (fp32, HW + 1 terms per sum) -> LayerNorm -> projection or MLP in fp32 against float64: the pooled row
    within 2^-16 (|n| + 1) |g| + HW u mean|x| rstd |g|, each projection layer within (K / 8 + 6) u (|row| @ |W|) plus
    the row's own bound through |W|; the normalised output within 2^-20 of its norm-1 values beyond that."""
    import torch
    import torch.nn.functional as F

    gen = torch.Generator().manual_seed(B * HW + C + mlp)
    x = torch.randn(B * HW, C, generator=gen).bfloat16().cuda()
    g = (1 + 0.2 * torch.randn(C, generator=gen)).cuda()
    b = (0.1 * torch.randn(C, generator=gen)).cuda()
    h = 2 * D
    w1T = (torch.randn(C, h, generator=gen) / math.sqrt(C)).cuda() if mlp else None
    b1 = (0.05 * torch.randn(h, generator=gen)).cuda() if mlp else None
    w2T = (torch.randn(h if mlp else C, D, generator=gen) / math.sqrt(h if mlp else C)).cuda()
    pooled, feat, out = head(x, HW, g, b, 1e-6, w1T, b1, w2T, D, 1)
    xd = x.double().view(B, HW, C)
    m_ = xd.mean(1)
    n = F.layer_norm(m_, (C,), None, None, 1e-6)
    rstd = 1.0 / torch.sqrt(m_.var(1, unbiased=False, keepdim=True) + 1e-6)
    pr = n * g.double() + b.double()
    e_p = 2.0 ** -16 * (n.abs() + 1) * g.double().abs() + (HW + 1) * U * xd.abs().mean(1) * rstd * g.double().abs() * 2
    _check(pooled, pr, e_p, "head pooled B=%d C=%d" % (B, C))

    def layer(row, e_row, WT, bias=None):
        K = WT.shape[0]
        y = row @ WT.double()
        if bias is not None:
            y = y + bias.double()
        e = (K / 8 + 6) * U * (row.abs() @ WT.double().abs()) + e_row @ WT.double().abs()
        return y, e

    if mlp:
        y1, e1 = layer(pr, e_p, w1T, b1)
        hd = 0.5 * y1 * (1 + torch.erf(y1 / math.sqrt(2)))
        e_h = e1 * 1.2 + 4 * U * hd.abs()   # gelu's slope is below 1.13
        f, e_f = layer(hd, e_h, w2T)
    else:
        f, e_f = layer(pr, e_p, w2T)
    _check(feat, f, e_f + 2 * U * f.abs(), "head feat mlp=%d B=%d C=%d" % (mlp, B, C))
    nf = f / f.norm(dim=1, keepdim=True)
    e_n = 2 * (e_f.norm(dim=1, keepdim=True) / f.norm(dim=1, keepdim=True)) + 2.0 ** -20
    _check(out, nf, e_n.expand_as(nf), "head out mlp=%d" % mlp)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("B,S", [(1, 224), (3, 256), (2, 320)])
def test_stem_patch_gemm_with_zero_k_tail(B, S):
    """im2col_patches at p = 4 into a zeroed [B (S/4)^2, 64] buffer writes columns 0..47 with the pixels (bf16, the
    conv weight's own flattening) and leaves 48..63 zero; the GEMM over all 64 columns with a zero-padded weight equals
    float64 conv2d(stride 4) of the same bf16 operands within the GEMM bound of test_gemm_gpu.py (K = 64)."""
    import torch
    import torch.nn.functional as F
    from clip_retrieval_b200._lib import lib, check

    gen = torch.Generator().manual_seed(S + B)
    px = torch.randn(B, 3, S, S, generator=gen).cuda()
    g = S // 4
    cols = torch.zeros(B * g * g, 64, dtype=torch.bfloat16, device="cuda")
    check(lib.b200_vision_front_bf16_device(px.data_ptr(), B, S, 4, 64, cols.data_ptr(), None, 0, 0, None, 0,
                                            _stream()), "vision_front")
    torch.cuda.synchronize()
    assert torch.count_nonzero(cols[:, 48:]) == 0
    want = px.bfloat16().view(B, 3, g, 4, g, 4).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, 48)
    assert torch.equal(cols[:, :48], want)
    C0 = 128
    w = (torch.randn(C0, 3, 4, 4, generator=gen) / math.sqrt(48)).bfloat16().cuda()
    wp = torch.zeros(C0, 64, dtype=torch.bfloat16, device="cuda")
    wp[:, :48] = w.reshape(C0, 48)
    bias = (0.02 * torch.randn(C0, generator=gen)).cuda()
    out = torch.empty(B * g * g, C0, dtype=torch.bfloat16, device="cuda")
    check(lib.b200_gemm_bf16_device(cols.data_ptr(), wp.data_ptr(), bias.data_ptr(), None, out.data_ptr(), B * g * g,
                                    C0, 64, 0, 0, _stream()), "gemm")
    torch.cuda.synchronize()
    xd = px.bfloat16().double()
    y = F.conv2d(xd, w.double(), bias.double(), stride=4).permute(0, 2, 3, 1).reshape(-1, C0)
    S_ = F.conv2d(xd.abs(), w.double().abs(), stride=4).permute(0, 2, 3, 1).reshape(-1, C0)
    e = (math.ceil(64 / 16) + 2) * 2.0 ** -22 * S_ + 2.0 ** -22 * y.abs()
    _check(out, y, 2.0 ** -8 * (y.abs() + e) + e, "stem gemm B=%d S=%d" % (B, S))


# ---- towers ------------------------------------------------------------------------------------------------------------

def _oracle_image(sd, arch, px):
    """oracle/convnext_ref.py in fp32 on the GPU, TF32 off for convolutions and matmuls."""
    import torch

    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        sd_dev = {k: v.cuda() for k, v in sd.items() if k.startswith("visual.")}
        return convnext_ref.encode_image(sd_dev, arch, px.cuda()).cpu().numpy()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
        torch.cuda.empty_cache()


def _images_apart(ref_i, what):
    from test_convnext_cpu import IMAGES_APART

    d = 1 - clip_ref.cosine(ref_i[0], ref_i[1])
    print("\n%s: images 1 - cos %.3g" % (what, d))
    assert d >= IMAGES_APART, (what, d)


def _check_tower(arch, sd, px, seed, what, discriminating=True):
    """encode_image / encode_text (raw) and embed_image (normalised) of px and seeded captions against the fp32
    oracles: 1 - cos <= 1e-3, norms within 2 %; the host entry stores the device entry's bits."""
    import clip_retrieval_b200 as m

    n = px.shape[0]
    model = m.B200Clip(arch, device=0, max_batch=n).load_state_dict(sd)
    tk = clip_ref.synth_tokens(n, arch, seed=seed)
    fi = model.encode_image(px.cuda()).cpu().numpy()
    ft = model.encode_text(tk.cuda()).cpu().numpy()
    ei = model.embed_image(px)
    assert np.array_equal(model.embed_image_device(px.cuda()).cpu().numpy(), ei)
    et = model.embed_text(tk)
    assert np.array_equal(model.embed_text_device(tk.cuda()).cpu().numpy(), et)
    del model
    ref_i = _oracle_image(sd, arch, px)
    ref_t = convnext_ref.encode_text(sd, arch, tk).numpy()
    if discriminating:
        _images_apart(ref_i, what)
    for kind, got, ref in (("image", fi, ref_i), ("text", ft, ref_t)):
        d = 1 - clip_ref.cosine(got, ref)
        print("\n%s %s: 1 - cos max %.3g" % (what, kind, d.max()))
        assert d.max() <= COS_TOL, (what, kind, d)
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), np.linalg.norm(ref, axis=1), rtol=2e-2)
    for got, ref in ((ei, ref_i), (et, ref_t)):
        n_ref = ref / np.linalg.norm(ref, axis=1, keepdims=True)
        assert (1 - clip_ref.cosine(got.astype(np.float32), n_ref)).max() <= COS_TOL
    return fi


def _check_case(case, arch=None):
    from test_convnext_cpu import tower_cases, tower_inputs

    a, sd, px = tower_inputs(case, arch=arch)
    _check_tower(a, sd, px, tower_cases()[case][1], case)


@pytest.mark.timeout(600)
def test_tiny_on_structured_images():
    _check_case("tiny")


@pytest.mark.timeout(600)
def test_tiny_matches_golden_and_oracle():
    """The golden's own inputs: pins the forward against transformers.ConvNextModel + open_clip's head."""
    import importlib.util

    import clip_retrieval_b200 as m

    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_convnext_golden", os.path.join(golden, "make_convnext_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    sd = m.synthetic_state_dict(gen.TINY, seed=0)
    fi = _check_tower(gen.TINY, sd, clip_ref.synth_images(gen.N, gen.TINY, seed=0), 0, "tiny golden",
                      discriminating=False)
    gold = np.load(os.path.join(golden, "clip_tiny-convnext.npz"))["image"]
    assert (1 - clip_ref.cosine(fi, gold)).max() <= COS_TOL


@pytest.mark.timeout(900)
@pytest.mark.parametrize("key", ["convnext_base", "convnext_base_w", "convnext_base_w_320", "convnext_large_d",
                                 "convnext_large_d_320", "convnext_xxlarge"])
def test_one_block_per_stage_at_real_widths(key):
    _check_case(key + "-1block")


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("key", ["convnext_base_w", "convnext_large_d_320"])
def test_full_depth_matches_oracle(key):
    """Full depth (3, 3, 27, 3) on the same weights' construction and structured images."""
    import clip_retrieval_b200 as m

    a = m.CONVNEXT_ARCHS["open_clip:" + key]
    _check_case(key + "-1block", arch=a)


@pytest.mark.timeout(600)
def test_batch1_graph_replay_is_bit_identical_to_eager_and_chunk_seams():
    """Batch 1 runs eagerly, is captured, then replayed: every call stores the same bits, as a handle with graphs off
    does.  Batch 5 on max_batch 2 runs in chunks 2, 2, 1 and equals those three calls made one by one."""
    import torch

    import clip_retrieval_b200 as m
    from test_convnext_cpu import tower_inputs

    a, sd, px = tower_inputs("convnext_large_d-1block", n=5)
    model = m.B200Clip(a, device=0, max_batch=2).load_state_dict(sd)
    one = px[:1].cuda()
    outs = [model.encode_image(one) for _ in range(4)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    assert torch.isfinite(outs[0]).all()
    five = model.encode_image(px.cuda())
    parts = torch.cat([model.encode_image(px[i:j].cuda()) for i, j in ((0, 2), (2, 4), (4, 5))])
    assert torch.equal(five, parts)
    assert torch.equal(five[:1], outs[0])
    del model
    prev = os.environ.get("B200_GRAPHS")
    os.environ["B200_GRAPHS"] = "0"   # read when the handle is created
    try:
        eager = m.B200Clip(a, device=0, max_batch=2).load_state_dict(sd)
    finally:
        if prev is None:
            del os.environ["B200_GRAPHS"]
        else:
            os.environ["B200_GRAPHS"] = prev
    for _ in range(3):
        assert torch.equal(eager.encode_image(one), outs[0])


# ---- drop-ins ----------------------------------------------------------------------------------------------------------

@pytest.mark.timeout(1500)
def test_load_clip_xxlarge_state_dict_file(tmp_path):
    """load_clip of `open_clip:convnext_xxlarge/laion2b_s34b_b82k_augreg_soup` from `<cache>/convnext_xxlarge-
    laion2b_s34b_b82k_augreg_soup.pt`, a full-size fp16 state_dict in open_clip's layout; its image features against
    the oracle on structured images."""
    import shutil

    import torch

    import clip_retrieval_b200 as m
    from test_resnet_cpu import structured_images

    name = "open_clip:convnext_xxlarge/laion2b_s34b_b82k_augreg_soup"
    a = m.CONVNEXT_ARCHS["open_clip:convnext_xxlarge"]
    sd = {k: v.half() for k, v in m.synthetic_state_dict(a, seed=4).items()}
    sd["logit_scale"] = torch.tensor(4.6052)
    torch.save(sd, str(tmp_path / "convnext_xxlarge-laion2b_s34b_b82k_augreg_soup.pt"))
    shutil.copy(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bpe_tiny.txt.gz"),
                str(tmp_path / "bpe_simple_vocab_16e6.txt.gz"))
    model, pre, tok = m.load_clip(name, warmup_batch_size=2, clip_cache_path=str(tmp_path))
    assert model.arch == a
    px = structured_images(2, a.image_size, seed=6)
    got = model.encode_image(px.cuda()).cpu().numpy()
    ref = _oracle_image({k: v.float() for k, v in sd.items()}, a, px)
    _images_apart(ref, "xxlarge.pt")
    d = 1 - clip_ref.cosine(got, ref)
    print("\nxxlarge.pt image: 1 - cos max %.3g" % d.max())
    assert d.max() <= COS_TOL
    t = model.embed_text(tok(["a photo of a cat", "a dog"]))
    assert t.shape == (2, 1024) and np.isfinite(t.astype(np.float32)).all()
    del model
    m.load_clip.cache_clear()
    torch.cuda.empty_cache()


@pytest.mark.timeout(900)
def test_mapper_rgb8_and_knn_service_on_large_d_320():
    """load_clip("synthetic:open_clip:convnext_large_d_320") -> ClipMapper: `image_rgb8` (the GPU transform at 320 px)
    stores the host transform's embeddings bit for bit, with max_batch 3 and 4 images (a ragged last chunk); then a
    B200KnnService text query on a 768-d index."""
    import torch

    import clip_retrieval_b200 as m
    from clip_retrieval_b200.model import SimpleTokenizer
    from oracle import synth_ref

    name = "synthetic:open_clip:convnext_large_d_320"
    mapper = m.ClipMapper(True, True, False, False, name, False, "", warmup_batch_size=3)
    a = mapper.model.arch
    assert a.image_size == 320 and mapper.model.max_batch == 3
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((360, 333), (200, 640), (320, 320), (500, 400))]
    tens = m.B200Preprocess(320)(imgs).cpu()
    tk = clip_ref.synth_tokens(4, a, seed=2)
    meta = {"image_filename": list("abcd"), "text": list("abcd")}
    out = mapper({"image_tensor": tens, "text_tokens": tk, **meta})
    assert out["image_embs"].shape == (4, 768) and out["text_embs"].shape == (4, 768)
    np.testing.assert_allclose(np.linalg.norm(out["image_embs"].astype(np.float32), axis=1), 1.0, atol=2e-3)
    via_rgb8 = mapper({"image_rgb8": imgs, "text_tokens": tk, **meta})["image_embs"]
    assert np.array_equal(via_rgb8, out["image_embs"])
    model = mapper.model
    d, n, k = 768, 3000, 20
    X = synth_ref.rows_f16(n, d, seed=5)
    idx = m.B200FlatIndex(d)
    idx.add(X)
    tok = SimpleTokenizer(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bpe_tiny.txt.gz"))
    res = m.ClipResource(model, tokenizer=tok, image_index=idx, text_index=idx)
    svc = m.B200KnnService({"cnx": res})
    got = svc.query(text_input="a photo of a cat", modality="image", num_images=k, num_result_ids=k, deduplicate=False)
    q = svc.compute_query_device(res, text_input="a photo of a cat")
    assert q.shape == (1, d) and abs(float(q.norm()) - 1.0) < 1e-3
    D, I = idx.search_device(q, k)
    assert [r["id"] for r in got] == [int(i) for i in I[0].cpu().numpy()]
    del svc, res, model, mapper
    m.load_clip.cache_clear()
    torch.cuda.empty_cache()
