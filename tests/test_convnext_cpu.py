"""The ConvNeXt CLIPs without a GPU: name resolution, the config table and parameter totals, a checkpoint round trip,
oracle/convnext_ref.py against the transformers golden, wrong forwards that the GPU tests' bar (1 - cos <= 1e-3
against the fp32 oracle) rejects, and a bf16 stand-in that shows how much of the bar a correct tower uses."""
import os
from dataclasses import replace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import clip_retrieval_b200 as m
from clip_retrieval_b200.model import resolve_arch
from oracle import clip_ref, convnext_ref
from test_resnet_cpu import structured_images

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COS_TOL = 1e-3   # test_convnext_gpu.py

# px, depths, dims, head, D, text (width, heads, layers), eps, pretrained tags, parameters (M, logit_scale included),
# image tower parameters (M, trunk + head)
TABLE = {
    "convnext_base": (224, (3, 3, 27, 3), (128, 256, 512, 1024), "linear", 512, (512, 8, 12), 1e-6,
                      ("laion400m_s13b_b51k",), 151.52, 88.09),
    "convnext_base_w": (256, (3, 3, 27, 3), (128, 256, 512, 1024), "linear", 640, (640, 10, 12), 1e-6,
                        ("laion2b_s13b_b82k", "laion2b_s13b_b82k_augreg", "laion_aesthetic_s13b_b82k"), 179.39, 88.22),
    "convnext_base_w_320": (320, (3, 3, 27, 3), (128, 256, 512, 1024), "linear", 640, (640, 10, 12), 1e-6,
                            ("laion_aesthetic_s13b_b82k", "laion_aesthetic_s13b_b82k_augreg"), 179.39, 88.22),
    "convnext_large_d": (256, (3, 3, 27, 3), (192, 384, 768, 1536), "mlp", 768, (768, 12, 16), 1e-6,
                         ("laion2b_s26b_b102k_augreg",), 351.77, 199.77),
    "convnext_large_d_320": (320, (3, 3, 27, 3), (192, 384, 768, 1536), "mlp", 768, (768, 12, 16), 1e-6,
                             ("laion2b_s29b_b131k_ft", "laion2b_s29b_b131k_ft_soup"), 351.77, 199.77),
    "convnext_xxlarge": (256, (3, 4, 30, 3), (384, 768, 1536, 3072), "linear", 1024, (1024, 16, 24), 1e-5,
                         ("laion2b_s34b_b82k_augreg", "laion2b_s34b_b82k_augreg_rewind",
                          "laion2b_s34b_b82k_augreg_soup"), 1200.58, 846.54),
}
SIX = tuple(TABLE)


def _names():
    out = []
    for k, row in TABLE.items():
        out.append(("open_clip:" + k, "open_clip:" + k, "open_clip:" + k))
        out.append(("synthetic:open_clip:" + k, "open_clip:" + k, "open_clip:" + k))
        for tag in row[7]:
            out.append(("open_clip:%s/%s" % (k, tag), "open_clip:" + k, "open_clip:%s/%s" % (k, tag)))
    return out


@pytest.mark.parametrize("name,table_key,key", _names())
def test_names_resolve(name, table_key, key):
    arch, got_key = resolve_arch(name)
    assert arch == m.CONVNEXT_ARCHS[table_key] and isinstance(arch, m.ConvNeXtArch) and not arch.quick_gelu
    assert got_key == key


@pytest.mark.parametrize("name", ["open_clip:convnext_base-quickgelu", "open_clip:convnext_base/openai",
                                  "open_clip:convnext_xxlarge-quickgelu/laion2b_s34b_b82k_augreg",
                                  "open_clip:convnext_large_d/laion2b_s29b_b131k_ft", "open_clip:convnext_tiny",
                                  "convnext_base"])
def test_refusals(name):
    with pytest.raises(ValueError):
        resolve_arch(name)


def test_tables_are_apart():
    others = set(m.ARCHS) | set(m.G14_ARCHS) | set(m.RESNET_ARCHS) | set(m.SIGLIP_ARCHS)
    assert not set(m.CONVNEXT_ARCHS) & others
    assert set(m.CONVNEXT_ARCHS) == {"open_clip:" + k for k in TABLE}
    assert all(not isinstance(a, m.ConvNeXtArch) for k, a in m.model.KNOWN_ARCHS.items() if k in others)


@pytest.mark.parametrize("key", SIX)
def test_configs_and_parameter_totals(key):
    px, depths, dims, head, D, (tw, th, tl), eps, tags, total, visual = TABLE[key]
    a = m.CONVNEXT_ARCHS["open_clip:" + key]
    assert (a.image_size, a.depths, a.dims, a.head_mlp, a.embed_dim, a.eps, a.tags) == (
        px, depths, dims, head == "mlp", D, eps, tags)
    assert (a.text.width, a.text.heads, a.text.layers, a.text.mlp, a.context_length, a.vocab_size) == (
        tw, th, tl, 4 * tw, 77, 49408)
    sd = m.synthetic_state_dict(a, seed=0)
    assert round((sum(v.numel() for v in sd.values()) + 1) / 1e6, 2) == total
    assert round(sum(v.numel() for k, v in sd.items() if k.startswith("visual.")) / 1e6, 2) == visual


def test_checkpoint_round_trip(tmp_path):
    """A state_dict saved in open_clip's layout (training-checkpoint wrapper, `module.` prefixes) reads back unchanged
    from `<cache>/<name>-<tag>.pt`."""
    from clip_retrieval_b200.model import _find_checkpoint, read_checkpoint

    name = "open_clip:convnext_large_d_320/laion2b_s29b_b131k_ft_soup"
    a, key = resolve_arch(name)
    a = replace(a, depths=(1, 1, 1, 1), text=m.Tower(a.text.width, 1, a.text.heads, a.text.mlp))
    sd = m.synthetic_state_dict(a, seed=1)
    torch.save({"epoch": 3, "state_dict": {"module." + k: v for k, v in sd.items()}},
               str(tmp_path / "convnext_large_d_320-laion2b_s29b_b131k_ft_soup.pt"))
    path = _find_checkpoint(key, str(tmp_path))
    assert path and path.endswith("convnext_large_d_320-laion2b_s29b_b131k_ft_soup.pt")
    back = read_checkpoint(path, a)
    assert set(back) == set(sd) and all(torch.equal(back[k], sd[k]) for k in sd)
    assert _find_checkpoint("open_clip:convnext_large_d_320", str(tmp_path)) is None


def _tiny():
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_convnext_golden", os.path.join(GOLDEN, "make_convnext_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    return gen


def test_oracle_matches_golden():
    gen = _tiny()
    sd = m.synthetic_state_dict(gen.TINY, seed=0)
    got = convnext_ref.encode_image(sd, gen.TINY, clip_ref.synth_images(gen.N, gen.TINY)).numpy()
    gold = np.load(os.path.join(GOLDEN, "clip_tiny-convnext.npz"))["image"]
    np.testing.assert_allclose(got, gold, rtol=1e-5, atol=1e-5 * np.abs(gold).max())


# ---- tower cases -------------------------------------------------------------------------------------------------------

def tower_cases():
    """name -> (arch, seed) of the tower checks on structured images, here against the wrong forwards and the bf16
    stand-in, and in test_convnext_gpu.py against the library: the tiny config, and each model at its real widths,
    image size and head with one block per stage (text tower cut to 2 layers)."""
    out = {"tiny": (_tiny().TINY, 1)}
    for k in SIX:
        a = m.CONVNEXT_ARCHS["open_clip:" + k]
        out[k + "-1block"] = (replace(a, depths=(1, 1, 1, 1), text=m.Tower(a.text.width, 2, a.text.heads, a.text.mlp)), 1)
    return out


CASES = ["tiny"] + [k + "-1block" for k in SIX]


def tower_inputs(case, n=2, arch=None):
    """(arch, weights, structured images) of a tower case; `arch` overrides the case's architecture."""
    a, seed = tower_cases()[case]
    a = arch or a
    return a, m.synthetic_state_dict(a, seed=seed), structured_images(n, a.image_size, seed=seed)


IMAGES_APART = 1e-2   # the least 1 - cos between the oracle's features of two images of a tower case


@pytest.mark.parametrize("case", CASES)
def test_tower_inputs_tell_images_apart(case):
    """On these inputs the features depend on the image: the oracle's two images differ by 1 - cos >= 1e-2, ten
    times the bar."""
    a, sd, px = tower_inputs(case)
    ref = convnext_ref.encode_image(sd, a, px).numpy()
    d = 1 - clip_ref.cosine(ref[0], ref[1])
    print("\n%s: images 1 - cos %.3g" % (case, d))
    assert d >= IMAGES_APART


# ---- wrong forwards ----------------------------------------------------------------------------------------------------

MUTATIONS = ["dw_taps_flipped", "gamma_dropped", "downsample_taps_transposed", "block_ln_skipped", "head_ln_skipped",
             "mean_is_pixel0", "gelu_dropped", "block_with_previous_weights", "head_gelu_dropped"]


@torch.no_grad()
def wrong_forward(sd, arch, px, mut=None):
    """convnext_ref's image forward with one named mistake (None: none).
    - dw_taps_flipped: the depthwise kernel applied as a convolution (taps flipped in both axes), not a correlation;
    - gamma_dropped: the blocks' layer scales not applied;
    - downsample_taps_transposed: every 2x2 downsample kernel read as w[..., j, i];
    - block_ln_skipped: fc1 reads the depthwise output without the block's LayerNorm;
    - head_ln_skipped: the pooled row goes to the head without head.norm;
    - mean_is_pixel0: the pooled row is pixel (0, 0) of the last map instead of its mean;
    - gelu_dropped: fc2 applied to fc1's output without the GELU between;
    - block_with_previous_weights: block 1 of stage 2 runs with block 0's weights (stage 2 gets 2 blocks for it);
    - head_gelu_dropped: the MLP head without its GELU (MLP heads only)."""
    sd = {k: v.float() for k, v in sd.items()}
    t, eps = "visual.trunk.", arch.eps
    x = convnext_ref.ln_channels(F.conv2d(px.float(), sd[t + "stem.0.weight"], sd[t + "stem.0.bias"], stride=4), sd,
                                 t + "stem.1", eps)
    for s, n in enumerate(arch.depths):
        p = "%sstages.%d." % (t, s)
        if s > 0:
            w = sd[p + "downsample.1.weight"]
            if mut == "downsample_taps_transposed":
                w = w.transpose(-1, -2)
            x = F.conv2d(convnext_ref.ln_channels(x, sd, p + "downsample.0", eps), w, sd[p + "downsample.1.bias"], stride=2)
        for j in range(n):
            b = "%sblocks.%d." % (p, j)
            if mut == "block_with_previous_weights" and s == 2 and j == 1:
                b = "%sblocks.0." % p
            C = x.shape[1]
            wdw = sd[b + "conv_dw.weight"]
            if mut == "dw_taps_flipped":
                wdw = wdw.flip(-1, -2)
            y = F.conv2d(x, wdw, sd[b + "conv_dw.bias"], padding=3, groups=C).permute(0, 2, 3, 1)
            if mut != "block_ln_skipped":
                y = F.layer_norm(y, (C,), sd[b + "norm.weight"], sd[b + "norm.bias"], eps)
            y = F.linear(y, sd[b + "mlp.fc1.weight"], sd[b + "mlp.fc1.bias"])
            if mut != "gelu_dropped":
                y = F.gelu(y)
            y = F.linear(y, sd[b + "mlp.fc2.weight"], sd[b + "mlp.fc2.bias"])
            if mut != "gamma_dropped":
                y = y * sd[b + "gamma"]
            x = x + y.permute(0, 3, 1, 2)
    pooled = x[:, :, 0, 0] if mut == "mean_is_pixel0" else x.mean((2, 3))
    if mut != "head_ln_skipped":
        pooled = F.layer_norm(pooled, (pooled.shape[1],), sd[t + "head.norm.weight"], sd[t + "head.norm.bias"], eps)
    if arch.head_mlp:
        h = F.linear(pooled, sd["visual.head.mlp.fc1.weight"], sd["visual.head.mlp.fc1.bias"])
        return F.linear(h if mut == "head_gelu_dropped" else F.gelu(h), sd["visual.head.mlp.fc2.weight"])
    return F.linear(pooled, sd["visual.head.proj.weight"])


@pytest.mark.parametrize("case", ["tiny", "convnext_base-1block", "convnext_large_d-1block"])
def test_restated_forward_is_the_oracle(case):
    a, sd, px = tower_inputs(case)
    np.testing.assert_allclose(wrong_forward(sd, a, px).numpy(), convnext_ref.encode_image(sd, a, px).numpy(),
                               rtol=1e-5, atol=1e-5)


WRONG_FLOOR = 2.8e-3   # about half the least 1 - cos measured over every case and mistake (see below)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("mut", MUTATIONS)
def test_wrong_forwards_fail_the_bar(case, mut):
    """On the synthetic weights and structured images (the GPU tests run the same inputs), against the fp32 oracle.
    Measured minimum 1 - cos: 5.7e-3 (convnext_base one block per stage, head LayerNorm skipped); the next closest
    mistake is the block LayerNorm skipped at 1.1e-2, every other one at 2.2e-2 or more.  The floor is 2.8 times the
    bar."""
    a = tower_cases()[case][0]
    if mut == "head_gelu_dropped" and not a.head_mlp:
        pytest.skip("linear head: no GELU to drop")
    if mut == "block_with_previous_weights" and a.depths[2] < 2:
        a = replace(a, depths=(a.depths[0], a.depths[1], 2, a.depths[3]))
    a, sd, px = tower_inputs(case, arch=a)
    ref = convnext_ref.encode_image(sd, a, px).numpy()
    bad = wrong_forward(sd, a, px, mut).numpy()
    d = 1 - clip_ref.cosine(bad, ref)
    print("\n%s %s: 1 - cos %s" % (case, mut, d))
    assert d.min() > WRONG_FLOOR, d


# ---- bf16 stand-in -----------------------------------------------------------------------------------------------------

@torch.no_grad()
def bf16_forward(sd, arch, px):
    """A correct forward in fp32 arithmetic that stores bf16 where the library does: the pixels (im2col), the GEMM
    weights (fc2 with gamma folded in fp64), the stem output and its LayerNorm, every dwconv7_ln output, the GELU hidden,
    the residual stream after each fc2 and downsample GEMM, and the ln_s2d rows.  The depthwise weights, the LayerNorm
    statistics and the head stay fp32."""
    sd = {k: v.double() for k, v in sd.items()}

    def bf(x):
        return x.float().bfloat16().float()

    t, eps = "visual.trunk.", arch.eps

    def ln_c(x, p):
        return bf(F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), sd[p + ".weight"].float(), sd[p + ".bias"].float(),
                               eps).permute(0, 3, 1, 2))

    x = bf(F.conv2d(bf(px), bf(sd[t + "stem.0.weight"]), sd[t + "stem.0.bias"].float(), stride=4))
    x = ln_c(x, t + "stem.1")
    for s, n in enumerate(arch.depths):
        p = "%sstages.%d." % (t, s)
        if s > 0:
            x = bf(F.conv2d(ln_c(x, p + "downsample.0"), bf(sd[p + "downsample.1.weight"]),
                            sd[p + "downsample.1.bias"].float(), stride=2))
        for j in range(n):
            b = "%sblocks.%d." % (p, j)
            C = x.shape[1]
            y = F.conv2d(x, sd[b + "conv_dw.weight"].float(), sd[b + "conv_dw.bias"].float(), padding=3, groups=C)
            y = bf(F.layer_norm(y.permute(0, 2, 3, 1), (C,), sd[b + "norm.weight"].float(), sd[b + "norm.bias"].float(),
                                eps))
            h = bf(F.gelu(F.linear(y, bf(sd[b + "mlp.fc1.weight"]), sd[b + "mlp.fc1.bias"].float())))
            g = sd[b + "gamma"]
            y = F.linear(h, bf(g[:, None] * sd[b + "mlp.fc2.weight"]), (g * sd[b + "mlp.fc2.bias"]).float())
            x = bf(x + y.permute(0, 3, 1, 2))
    pooled = x.mean((2, 3))
    pooled = F.layer_norm(pooled, (pooled.shape[1],), sd[t + "head.norm.weight"].float(),
                          sd[t + "head.norm.bias"].float(), eps)
    return convnext_ref.head({k: v.float() for k, v in sd.items()}, arch, pooled)


STAND_IN_SHARE = 0.1   # a correct bf16 forward uses at most this share of the bar on every case


@pytest.mark.parametrize("case", CASES)
def test_bf16_stand_in_stays_inside_the_bar(case):
    """The rounding a correct bf16 forward carries on these inputs is well inside the bar: at most a tenth of it.
    Measured: 4.3e-5 tiny (4 % of the bar), 6e-6 - 1e-5 at real widths (1 %)."""
    a, sd, px = tower_inputs(case)
    ref = convnext_ref.encode_image(sd, a, px).numpy()
    d = 1 - clip_ref.cosine(bf16_forward(sd, a, px).numpy(), ref)
    print("\n%s: bf16 stand-in 1 - cos %s (%.2f of the bar)" % (case, d, d.max() / COS_TOL))
    assert d.max() <= COS_TOL * STAND_IN_SHARE, d
