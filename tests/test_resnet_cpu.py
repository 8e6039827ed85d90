"""The ResNet CLIPs without a GPU: name resolution, the config table and parameter totals, oracle/resnet_ref.py against
the torch.nn golden, and wrong forwards that the GPU tests' bar (1 - cos <= 1e-3 against the fp32 oracle) rejects."""
import os
from dataclasses import replace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import clip_retrieval_b200 as m
from oracle import clip_ref, resnet_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3   # test_resnet_gpu.py

# (layers, width, image px, embed_dim, text width / heads / layers, T of the attention pool, parameters in millions as
# open_clip's model profile lists them, recalled)
TABLE = {
    "RN50": ((3, 4, 6, 3), 64, 224, 1024, (512, 8, 12), 50, 102.0),
    "RN101": ((3, 4, 23, 3), 64, 224, 512, (512, 8, 12), 50, 119.7),
    "RN50x4": ((4, 6, 10, 6), 80, 288, 640, (640, 10, 12), 82, 178.3),
    "RN50x16": ((6, 8, 18, 8), 96, 384, 768, (768, 12, 12), 145, 291.0),
    "RN50x64": ((3, 15, 36, 10), 128, 448, 1024, (1024, 16, 12), 197, 623.3),
}


@pytest.mark.parametrize("name,key,quick", [
    ("RN50", "RN50", True), ("RN101", "RN101", True), ("RN50x4", "RN50x4", True), ("RN50x16", "RN50x16", True),
    ("RN50x64", "RN50x64", True),
    ("open_clip:RN50", "open_clip:RN50", False), ("open_clip:RN50/openai", "open_clip:RN50", True),
    ("open_clip:RN50/yfcc15m", "open_clip:RN50", False), ("open_clip:RN50/cc12m", "open_clip:RN50", False),
    ("open_clip:RN50-quickgelu/yfcc15m", "open_clip:RN50", True), ("open_clip:RN50-quickgelu/cc12m", "open_clip:RN50", True),
    ("open_clip:RN101/openai", "open_clip:RN101", True), ("open_clip:RN101/yfcc15m", "open_clip:RN101", False),
    ("open_clip:RN101-quickgelu/yfcc15m", "open_clip:RN101", True),
    ("open_clip:RN50x4/openai", "open_clip:RN50x4", True), ("open_clip:RN50x16/openai", "open_clip:RN50x16", True),
    ("open_clip:RN50x64/openai", "open_clip:RN50x64", True), ("synthetic:RN50x64", "RN50x64", True),
    ("synthetic:open_clip:RN101-quickgelu", "open_clip:RN101", True),
])
def test_names_resolve(name, key, quick):
    from clip_retrieval_b200.model import resolve_arch

    arch, _ = resolve_arch(name)
    assert arch == replace(m.RESNET_ARCHS[key], quick_gelu=quick)
    assert isinstance(arch, m.ResNetArch)


def test_tables_are_apart():
    assert not set(m.RESNET_ARCHS) & (set(m.ARCHS) | set(m.G14_ARCHS))
    assert all(isinstance(a, m.ClipArch) for a in list(m.ARCHS.values()) + list(m.G14_ARCHS.values()))
    assert set(m.RESNET_ARCHS) == set(TABLE) | {"open_clip:" + k for k in TABLE}
    with pytest.raises(ValueError):
        from clip_retrieval_b200.model import resolve_arch

        resolve_arch("RN152")


@pytest.mark.parametrize("key", sorted(TABLE))
def test_configs_and_parameter_totals(key):
    layers, w, px, D, (tw, th, tl), T, millions = TABLE[key]
    for name, quick in ((key, True), ("open_clip:" + key, False)):
        a = m.RESNET_ARCHS[name]
        assert (a.layers, a.width, a.image_size, a.embed_dim, a.quick_gelu) == (layers, w, px, D, quick)
        assert (a.text.width, a.text.heads, a.text.layers, a.text.mlp) == (tw, th, tl, 4 * tw)
        assert a.heads == 32 * w // 64 and (a.image_size // 32) ** 2 + 1 == T
    sd = m.synthetic_state_dict(m.RESNET_ARCHS[key], seed=0)
    # parameters: everything but the BatchNorm buffers, + logit_scale (not in the synthetic state_dict)
    n = sum(v.numel() for k, v in sd.items() if not k.endswith(("running_mean", "running_var", "num_batches_tracked")))
    assert round((n + 1) / 1e6, 1) == millions
    assert sd["visual.attnpool.positional_embedding"].shape == (T, 32 * w)


def _tiny():
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_rn_golden", os.path.join(GOLDEN, "make_rn_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    return gen


def test_oracle_matches_golden():
    gen = _tiny()
    sd = m.synthetic_state_dict(gen.TINY, seed=0)
    got = resnet_ref.encode_image(sd, gen.TINY, clip_ref.synth_images(gen.N, gen.TINY)).numpy()
    gold = np.load(os.path.join(GOLDEN, "clip_tiny-rn.npz"))["image"]
    np.testing.assert_allclose(got, gold, rtol=1e-5, atol=1e-5 * np.abs(gold).max())


# ---- wrong forwards ----------------------------------------------------------------------------------------------------

MUTATIONS = ["bn_left_out", "pool_before_conv2", "downsample_without_pool", "no_mean_token", "taps_transposed",
             "relu_before_add", "block_with_previous_weights"]


@torch.no_grad()
def wrong_forward(sd, arch, px, mut=None):
    """resnet_ref's image forward with one named mistake (None: none).
    - bn_left_out: every convolution's weight used as is, BatchNorm not applied (no fold);
    - pool_before_conv2: a strided block pools before its 3x3 convolution instead of after;
    - downsample_without_pool: the identity branch subsamples (a strided 1x1 convolution) instead of averaging;
    - no_mean_token: the attention pool runs on the pixels alone (token 0 = the first pixel);
    - taps_transposed: every 3x3 kernel read as w[..., s, r];
    - relu_before_add: relu(conv3 branch) + identity;
    - block_with_previous_weights: block 2 of stage 2 (layer2.2) runs with block 1's weights (layer2.1).  Stages of
      one block have no two blocks of the same shapes, so on those configs stage 2 is given 3 blocks for this one."""
    sd = {k: v.float() for k, v in sd.items()}
    relu = F.relu

    def cbn(x, conv, bn, stride=1, padding=0):
        w = sd[conv + ".weight"]
        if mut == "taps_transposed" and w.shape[-1] == 3:
            w = w.transpose(-1, -2)
        y = F.conv2d(x, w, stride=stride, padding=padding)
        return y if mut == "bn_left_out" else resnet_ref._bn(y, sd, bn)

    x = relu(cbn(px.float(), "visual.conv1", "visual.bn1", 2, 1))
    x = relu(cbn(x, "visual.conv2", "visual.bn2", 1, 1))
    x = F.avg_pool2d(relu(cbn(x, "visual.conv3", "visual.bn3", 1, 1)), 2)
    for s, n in enumerate(arch.layers):
        for j in range(n):
            p = "visual.layer%d.%d." % (s + 1, j)
            wp = "visual.layer2.1." if (mut == "block_with_previous_weights" and s == 1 and j == 2) else p
            stride = 2 if (j == 0 and s > 0) else 1
            out = relu(cbn(x, wp + "conv1", wp + "bn1"))
            if stride > 1 and mut == "pool_before_conv2":
                out = F.avg_pool2d(out, stride)
            out = relu(cbn(out, wp + "conv2", wp + "bn2", 1, 1))
            if stride > 1 and mut != "pool_before_conv2":
                out = F.avg_pool2d(out, stride)
            out = cbn(out, wp + "conv3", wp + "bn3")
            idn = x
            if (p + "downsample.0.weight") in sd:
                if stride > 1:
                    idn = idn[:, :, ::stride, ::stride] if mut == "downsample_without_pool" else F.avg_pool2d(idn, stride)
                idn = cbn(idn, p + "downsample.0", p + "downsample.1")
            x = relu(out) + idn if mut == "relu_before_add" else relu(out + idn)
    heads = 32 * arch.width // 64
    if mut != "no_mean_token":
        return resnet_ref.attnpool(sd, x, heads)
    a = "visual.attnpool."
    B, C = x.shape[:2]
    t = x.flatten(2).permute(0, 2, 1) + sd[a + "positional_embedding"][1:]
    q = (t[:, :1] @ sd[a + "q_proj.weight"].t() + sd[a + "q_proj.bias"]).view(B, 1, heads, 64).transpose(1, 2)
    k = (t @ sd[a + "k_proj.weight"].t() + sd[a + "k_proj.bias"]).view(B, -1, heads, 64).transpose(1, 2)
    v = (t @ sd[a + "v_proj.weight"].t() + sd[a + "v_proj.bias"]).view(B, -1, heads, 64).transpose(1, 2)
    o = (torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1) @ v).transpose(1, 2).reshape(B, C)
    return o @ sd[a + "c_proj.weight"].t() + sd[a + "c_proj.bias"]


def structured_images(n, S, seed):
    """Images that differ in their coarse content: a bilinear 4 x 4 random field + fine noise, in the preprocess range.
    (clip_ref.synth_images are i.i.d. noise, statistically alike: a ResNet's pooled features of any two of them agree
    to 1 - cos ~ 1e-4, so a wrong forward can sit inside the bar.)"""
    g = torch.Generator().manual_seed(3000 + seed)
    low = torch.randn(n, 3, 4, 4, generator=g)
    x = F.interpolate(low, size=(S, S), mode="bilinear", align_corners=False) + 0.3 * torch.randn(n, 3, S, S, generator=g)
    return x.clamp(-1.80, 2.15)


def sensitise(sd, qk, pos):
    """The synthetic weights with a sharper attention pool: q / k projections x qk, positional embedding x pos, so that
    the query token and the pixels it picks show in the output (a documented transform, as tests/tower_ref.py uses).
    The sharper the softmax, the more it also amplifies the forward's bf16 rounding (bf16_forward below): x 8 / x 20
    puts a correct bf16 forward at 1 - cos 1.2e-3 (RN50x4, one block per stage) to 2.5e-3 (RN50 full depth)."""
    sd = dict(sd)
    for n in ("q", "k"):
        sd["visual.attnpool.%s_proj.weight" % n] = sd["visual.attnpool.%s_proj.weight" % n] * qk
    sd["visual.attnpool.positional_embedding"] = sd["visual.attnpool.positional_embedding"] * pos
    return sd


FIVE = ("RN50", "RN101", "RN50x4", "RN50x16", "RN50x64")


def tower_cases():
    """name -> (arch, seed, (qk, pos) of sensitise) of the tower checks that run on structured images, here against the
    wrong forwards and the bf16 stand-in, and in test_resnet_gpu.py against the library: the tiny config and each
    model at its real widths, image size and heads with one block per stage (text tower cut to 2 layers), on q / k x 2
    and positions x 10; full-depth RN50 and RN50x4 on the plain weights, which at depth tell images apart on their
    own (sharpening the pool there lifts the bf16 stand-in to 9e-4 - 4e-3)."""
    out = {"tiny": (_tiny().TINY, 1, (2, 10))}
    for k in FIVE:
        a = m.RESNET_ARCHS[k]
        out[k + "-1block"] = (replace(a, layers=(1, 1, 1, 1), text=m.Tower(a.text.width, 2, a.text.heads, a.text.mlp)),
                              1, (2, 10))
    for k in ("RN50", "RN50x4"):
        out[k + "-full"] = (m.RESNET_ARCHS[k], 2, (1, 1))
    return out


CASES = ["tiny"] + [k + "-1block" for k in FIVE] + ["RN50-full", "RN50x4-full"]


def tower_inputs(case, n=2, arch=None):
    """(arch, weights, structured images) of a tower case; `arch` overrides the case's architecture."""
    a, seed, (qk, pos) = tower_cases()[case]
    a = arch or a
    return a, sensitise(m.synthetic_state_dict(a, seed=seed), qk, pos), structured_images(n, a.image_size, seed=seed)


IMAGES_APART = 1e-2   # the least 1 - cos between the oracle's features of two images of a tower case


@pytest.mark.parametrize("case", CASES)
def test_tower_inputs_tell_images_apart(case):
    """On these inputs the features depend on the image: the oracle's two images differ by 1 - cos >= 1e-2, ten
    times the bar (measured 0.025 tiny, 0.058 - 0.116 at real widths)."""
    a, sd, px = tower_inputs(case)
    ref = resnet_ref.encode_image(sd, a, px).numpy()
    d = 1 - clip_ref.cosine(ref[0], ref[1])
    print("\n%s: images 1 - cos %.3g" % (case, d))
    assert d >= IMAGES_APART


@pytest.mark.parametrize("case", ["tiny", "RN50-1block", "RN50x4-full"])
def test_restated_forward_is_the_oracle(case):
    a, sd, px = tower_inputs(case)
    np.testing.assert_allclose(wrong_forward(sd, a, px).numpy(), resnet_ref.encode_image(sd, a, px).numpy(),
                               rtol=1e-5, atol=1e-5)


@torch.no_grad()
def bf16_forward(sd, arch, px):
    """A correct forward in fp32 arithmetic that stores bf16 where the library does: the folded weights (fp64 fold),
    every convolution / GEMM output after its epilogue (bias, residual, ReLU in fp32), the pools, the attention-pool
    tokens, q / k / v, the unnormalised probabilities before P·V and the attention output; c_proj in fp32."""
    sd = {k: v.double() for k, v in sd.items()}

    def bf(x):
        return x.bfloat16().float()

    def cbn(x, conv, bn, stride=1, padding=0, relu=True, res=None):
        sc = sd[bn + ".weight"] / torch.sqrt(sd[bn + ".running_var"] + 1e-5)
        w = bf((sd[conv + ".weight"] * sc[:, None, None, None]).float())
        y = F.conv2d(x, w, stride=stride, padding=padding) + (sd[bn + ".bias"] - sd[bn + ".running_mean"] * sc).float()[
            None, :, None, None]
        if res is not None:
            y = y + res
        return bf(F.relu(y) if relu else y)

    x = cbn(bf(px.float()), "visual.conv1", "visual.bn1", 2, 1)
    x = cbn(x, "visual.conv2", "visual.bn2", 1, 1)
    x = bf(F.avg_pool2d(cbn(x, "visual.conv3", "visual.bn3", 1, 1), 2))
    for s, n in enumerate(arch.layers):
        for j in range(n):
            p = "visual.layer%d.%d." % (s + 1, j)
            stride = 2 if (j == 0 and s > 0) else 1
            out = cbn(cbn(x, p + "conv1", p + "bn1"), p + "conv2", p + "bn2", 1, 1)
            if stride > 1:
                out = bf(F.avg_pool2d(out, stride))
            idn = x
            if p + "downsample.0.weight" in sd:
                xi = bf(F.avg_pool2d(x, stride)) if stride > 1 else x
                idn = cbn(xi, p + "downsample.0", p + "downsample.1", relu=False)
            x = cbn(out, p + "conv3", p + "bn3", res=idn)
    a = "visual.attnpool."
    B, C = x.shape[:2]
    h = C // 64
    t = x.flatten(2).permute(0, 2, 1)
    t = bf(torch.cat([t.mean(1, keepdim=True), t], 1) + sd[a + "positional_embedding"].float())

    def proj(n):
        return bf(t @ bf(sd[a + n + "_proj.weight"].float()).t() + sd[a + n + "_proj.bias"].float())

    q = proj("q")[:, :1].view(B, 1, h, 64).transpose(1, 2)
    k = proj("k").view(B, -1, h, 64).transpose(1, 2)
    v = proj("v").view(B, -1, h, 64).transpose(1, 2)
    sc = (q @ k.transpose(-1, -2)) / 8.0
    pr = torch.exp(sc - sc.amax(-1, keepdim=True))
    o = bf((bf(pr) @ v) / pr.sum(-1, keepdim=True)).transpose(1, 2).reshape(B, C)
    return o @ bf(sd[a + "c_proj.weight"].float()).t() + sd[a + "c_proj.bias"].float()


@pytest.mark.parametrize("case", CASES)
def test_bf16_stand_in_stays_inside_the_bar(case):
    """The rounding a correct bf16 forward carries on these inputs is well inside the bar: at most half of it
    (measured at most 3.1e-4, RN50 full depth).  Under the sharper x 8 / x 20 pool the same stand-in reaches
    1.2e-3 - 2.5e-3, as the library did on it: that is why the cases use x 2 / x 10 and, at full depth, none."""
    a, sd, px = tower_inputs(case)
    ref = resnet_ref.encode_image(sd, a, px).numpy()
    d = 1 - clip_ref.cosine(bf16_forward(sd, a, px).numpy(), ref)
    print("\n%s: bf16 stand-in 1 - cos %s" % (case, d))
    assert d.max() <= COS_TOL / 2, d


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("mut", MUTATIONS)
def test_wrong_forwards_fail_the_bar(case, mut):
    """On the sensitised weights and structured images (the GPU tests run the same inputs), against the fp32 oracle.
    Measured minimum 1 - cos: 3.9e-3 (tiny, taps transposed); at real widths 4.1e-3 (RN50x64 one block per stage, pool
    before conv2 and taps transposed), at full depth 1.2e-2."""
    a = tower_cases()[case][0]
    if mut == "block_with_previous_weights" and a.layers[1] < 3:
        a = replace(a, layers=(a.layers[0], 3) + tuple(a.layers[2:]))
    a, sd, px = tower_inputs(case, arch=a)
    ref = resnet_ref.encode_image(sd, a, px).numpy()
    bad = wrong_forward(sd, a, px, mut).numpy()
    d = 1 - clip_ref.cosine(bad, ref)
    print("\n%s %s: 1 - cos %s" % (case, mut, d))
    assert d.min() > COS_TOL, d
