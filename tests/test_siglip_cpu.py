"""SigLIP without a GPU: name resolution, the model table against its parameter counts, the checkpoint round trip,
the tokenizer against transformers' PreTrainedTokenizerFast under open_clip's call arguments, the squash transform
with mean = std = 0.5, the fp32 oracle (tests/siglip_ref.py) against transformers' SiglipModel, and the inputs on
which the GPU tower tests can fail.  The file takes about 20 s on 8 CPU cores."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import clip_retrieval_b200 as m
import siglip_ref
from clip_retrieval_b200.model import (preprocess_params, read_checkpoint, resolve_arch, siglip_clean, siglip_tokenizer,
                                       synthetic_state_dict)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# (total, vision, text) parameters, millions, of open_clip's model profile (DESIGN.md §5 (xix))
PARAMS = {
    "ViT-B-16-SigLIP": (203.16, 92.88, 110.27),
    "ViT-B-16-SigLIP-256": (203.20, 92.93, 110.27),
    "ViT-B-16-SigLIP-384": (203.45, 93.18, 110.27),
    "ViT-B-16-SigLIP-512": (203.79, 93.52, 110.27),
    "ViT-B-16-SigLIP-i18n-256": (370.63, 92.93, 277.70),
    "ViT-L-16-SigLIP-256": (652.15, 315.96, 336.19),
    "ViT-L-16-SigLIP-384": (652.48, 316.28, 336.19),
    "ViT-SO400M-14-SigLIP": (877.36, 427.68, 449.68),
    "ViT-SO400M-14-SigLIP-384": (877.96, 428.23, 449.73),
}
# name -> (image tokens, head dim, context)
SHAPES = {"ViT-B-16-SigLIP": (196, 64, 64), "ViT-B-16-SigLIP-256": (256, 64, 64), "ViT-B-16-SigLIP-384": (576, 64, 64),
          "ViT-B-16-SigLIP-512": (1024, 64, 64), "ViT-B-16-SigLIP-i18n-256": (256, 64, 64),
          "ViT-L-16-SigLIP-256": (256, 64, 64), "ViT-L-16-SigLIP-384": (576, 64, 64),
          "ViT-SO400M-14-SigLIP": (256, 72, 16), "ViT-SO400M-14-SigLIP-384": (729, 72, 64)}


def golden_module():
    spec = importlib.util.spec_from_file_location("make_siglip_golden", os.path.join(GOLDEN, "make_siglip_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def tiny_arch():
    g = golden_module()
    t = m.Tower(g.W, g.LAYERS, g.HEADS, g.MLP)
    return m.SigLIPArch(g.W, g.S, g.P, t, t, context_length=g.CTX, vocab_size=g.VOCAB)


def cos_dist(a, b):
    a, b = torch.as_tensor(np.asarray(a, dtype=np.float64)), torch.as_tensor(np.asarray(b, dtype=np.float64))
    return (1 - F.cosine_similarity(a, b, dim=-1)).numpy()


def structured_images(n, S, seed):
    """A bilinear 4 x 4 random field + fine noise (as tests/test_resnet_cpu.py): images that differ in coarse content."""
    g = torch.Generator().manual_seed(3000 + seed)
    low = torch.randn(n, 3, 4, 4, generator=g)
    x = F.interpolate(low, size=(S, S), mode="bilinear", align_corners=False) + 0.3 * torch.randn(n, 3, S, S, generator=g)
    return x.clamp(-1.0, 1.0)


def captions(n, arch, seed):
    """Token rows of different lengths: words, </s> (id 1), then pads (id 1), as the tokenizer writes them."""
    g = torch.Generator().manual_seed(4000 + seed)
    ids = torch.ones(n, arch.context_length, dtype=torch.long)
    for i in range(n):
        L = 2 + (i * 5) % max(1, arch.context_length - 3)
        ids[i, :L] = torch.randint(3, arch.vocab_size, (L,), generator=g)
    return ids


# ---- names and the table ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(PARAMS))
def test_names_resolve(name):
    for spelled in ("open_clip:" + name, "open_clip:%s/webli" % name, "synthetic:open_clip:%s/webli" % name):
        arch, key = resolve_arch(spelled)
        assert arch is m.SIGLIP_ARCHS["open_clip:" + name] and key == "open_clip:" + name
    for bad in ("open_clip:%s-quickgelu" % name, "open_clip:%s/openai" % name, "open_clip:%s-quickgelu/webli" % name):
        with pytest.raises(ValueError, match="SigLIP"):
            resolve_arch(bad)
    assert preprocess_params("open_clip:%s/webli" % name) == ("squash", (0.5,) * 3, (0.5,) * 3)
    assert preprocess_params("synthetic:open_clip:" + name)[0] == "squash"


def test_other_transforms_unchanged():
    assert preprocess_params("ViT-B/32") == ("shortest", m.model.OPENAI_MEAN, m.model.OPENAI_STD)
    assert preprocess_params("open_clip:ViT-H-14-378-quickgelu/dfn5b")[0] == "squash"
    assert preprocess_params("open_clip:ViT-H-14-378-quickgelu/dfn5b")[1] == m.model.OPENAI_MEAN


@pytest.mark.parametrize("name", sorted(PARAMS))
def test_table_figures(name):
    arch = m.SIGLIP_ARCHS["open_clip:" + name]
    T, hd, ctx = SHAPES[name]
    assert (arch.image_size // arch.patch) ** 2 == T and arch.vision.width // arch.vision.heads == hd
    assert arch.context_length == ctx and arch.embed_dim == arch.vision.width == arch.text.width
    with torch.device("meta"):
        sd = synthetic_state_dict(arch)
    vis = sum(v.numel() for k, v in sd.items() if k.startswith("visual."))
    txt = sum(v.numel() for k, v in sd.items() if k.startswith("text."))
    assert len(sd) == sum(1 for k in sd if k.startswith(("visual.", "text.")))
    assert (round((vis + txt) / 1e6, 2), round(vis / 1e6, 2), round(txt / 1e6, 2)) == PARAMS[name]


def test_checkpoint_round_trip(tmp_path):
    arch = tiny_arch()
    sd = synthetic_state_dict(arch, seed=3)
    path = str(tmp_path / "ViT-B-16-SigLIP.bin")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, path)
    back = read_checkpoint(path, arch)
    assert sorted(back) == sorted(sd) and all(torch.equal(back[k], sd[k]) for k in sd)


# ---- tokenizer ------------------------------------------------------------------------------------------------------

def tiny_tokenizer_json(path):
    """A Unigram tokenizer with SigLIP's shape: <pad> 0, </s> 1, <unk> 2, a Metaspace pre-tokenizer and a `$A </s>`
    post-processor."""
    from tokenizers import Tokenizer, models, pre_tokenizers, decoders, processors

    words = ["a", "photo", "of", "the", "cat", "dog", "on", "red", "blue", "car", "x", "y", "z"]
    vocab = [("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0), ("▁", -2.0)]
    vocab += [("▁" + w, -3.0 - 0.1 * i) for i, w in enumerate(words)]
    vocab += [(c, -6.0) for c in "abcdefghijklmnopqrstuvwxyz0123456789"]
    tok = Tokenizer(models.Unigram(vocab, unk_id=2, byte_fallback=False))
    tok.pre_tokenizer = pre_tokenizers.Metaspace()
    tok.decoder = decoders.Metaspace()
    tok.post_processor = processors.TemplateProcessing(single="$A </s>", special_tokens=[("</s>", 1)])
    tok.save(path)


TEXTS = ["A photo of the cat.", "a_photo_of_the_DOG!!", "  red   car,  blue car; (x-y-z)  ", "Photo",
         " ".join(["cat"] * 30), "", "a photo of the red dog on the blue car x y z"]


def test_clean_is_canonicalize():
    assert siglip_clean("A_b, C!  d") == "a b c d"
    assert siglip_clean("  Hello,\tWORLD...  ") == "hello world"
    assert siglip_clean("x-y_z") == "xy z"


def test_tokenizer_matches_transformers(tmp_path):
    from transformers import PreTrainedTokenizerFast

    arch = m.SIGLIP_ARCHS["open_clip:ViT-SO400M-14-SigLIP"]      # context 16: the 30-word text is truncated
    folder = tmp_path / arch.tokenizer
    folder.mkdir(parents=True)
    tiny_tokenizer_json(str(folder / "tokenizer.json"))
    ours = siglip_tokenizer(arch, str(tmp_path))(TEXTS)
    hf = PreTrainedTokenizerFast(tokenizer_file=str(folder / "tokenizer.json"), pad_token="</s>", eos_token="</s>",
                                 unk_token="<unk>")
    want = hf([siglip_clean(t) for t in TEXTS], max_length=arch.context_length, padding="max_length",
              truncation=True, return_tensors="pt").input_ids
    assert ours.shape == (len(TEXTS), 16) and torch.equal(ours, want)
    assert int(ours[4, -1]) == 1 and int(ours[0, 0]) != 1
    missing = siglip_tokenizer(arch, str(tmp_path / "nowhere"))
    with pytest.raises(RuntimeError, match="tokenizer"):
        missing(["x"])


# ---- transform ------------------------------------------------------------------------------------------------------

def _ref_images():
    from PIL import Image

    folder = os.path.join(GOLDEN, "ref_images")
    names = sorted(os.listdir(folder))
    assert names
    return [Image.open(os.path.join(folder, n)) for n in names]


def test_squash_transform_matches_pillow_and_hf():
    from torchvision import transforms as T
    from torchvision.transforms import InterpolationMode
    from transformers import SiglipImageProcessor

    from PIL import Image

    mode, mean, std = preprocess_params("open_clip:ViT-B-16-SigLIP/webli")
    ours = m.model.make_preprocess(224, mode, mean, std)
    hf = SiglipImageProcessor(size={"height": 224, "width": 224}, resample=Image.BICUBIC, image_mean=list(mean),
                              image_std=list(std), do_rescale=True, rescale_factor=1 / 255)
    for im in _ref_images():
        rgb = im.convert("RGB")
        x = ours(im)
        want = T.Normalize(mean, std)(T.ToTensor()(rgb.resize((224, 224), Image.BICUBIC)))
        assert torch.equal(x, want)
        assert torch.equal(x, T.Compose([T.Resize((224, 224), interpolation=InterpolationMode.BICUBIC),
                                         T.ToTensor(), T.Normalize(mean, std)])(rgb))
        # transformers resizes through its own path: the same bicubic squash, but a pixel can land one 8-bit level
        # (2/255 after the 0.5 / 0.5 normalisation) away where the resampled value sits near a rounding boundary
        h = torch.as_tensor(np.asarray(hf(rgb, return_tensors="np")["pixel_values"][0]))
        d = (h - x).abs()
        assert float(d.max()) <= 2 / 255 + 1e-6 and float((d > 1e-5).float().mean()) <= 0.01


# ---- the oracle -----------------------------------------------------------------------------------------------------

def test_oracle_matches_transformers_golden():
    g = golden_module()
    arch = tiny_arch()
    sd = g.state_dict()
    px, ids = g.inputs()
    gold = np.load(os.path.join(GOLDEN, "siglip_tiny.npz"))
    with torch.no_grad():
        img = siglip_ref.image_features(sd, arch, px).numpy()
        txt = siglip_ref.text_features(sd, arch, ids).numpy()
    assert np.abs(img - gold["image"]).max() <= 1e-5 * max(1.0, np.abs(gold["image"]).max())
    assert np.abs(txt - gold["text"]).max() <= 1e-5 * max(1.0, np.abs(gold["text"]).max())


# ---- sensitivity: inputs on which the GPU tower bar (1 - cos <= 1e-3) can fail ----------------------------------------

COS_TOL = 1e-3
# the wrong forwards below land at least this far above the bar on the tower cases: about half the smallest measured,
# 3.8e-3 (the positional table shifted one row on the 2-layer SO400M case)
FLOOR = 1.9


def sensitivity_cases():
    """(name, arch, state_dict): the tiny golden model and two table entries cut to 2 layers, sensitised."""
    g = golden_module()
    out = [("tiny", tiny_arch(), g.state_dict())]
    from dataclasses import replace

    for key in ("open_clip:ViT-B-16-SigLIP", "open_clip:ViT-SO400M-14-SigLIP"):
        a = m.SIGLIP_ARCHS[key]
        a = replace(a, vision=replace(a.vision, layers=2), text=replace(a.text, layers=2), vocab_size=1000)
        out.append((key, a, synthetic_state_dict(a, seed=1)))
    return [(n, a, sensitise(sd)) for n, a, sd in out]


def sensitise(sd):
    """A documented transform that lets a dropped latent-q bias and a shifted positional row rise above bf16 noise on
    random weights: pos_embed x 8, attn_pool.q.bias x 40, attn_pool.q.weight x 3 (a sharper pool)."""
    sd = dict(sd)
    sd["visual.trunk.pos_embed"] = sd["visual.trunk.pos_embed"] * 8
    sd["visual.trunk.attn_pool.q.bias"] = sd["visual.trunk.attn_pool.q.bias"] * 40
    sd["visual.trunk.attn_pool.q.weight"] = sd["visual.trunk.attn_pool.q.weight"] * 3
    return sd


def _mutated_sd(sd, what):
    sd = dict(sd)
    if what == "patch_bias_dropped":
        sd["visual.trunk.patch_embed.proj.bias"] = torch.zeros_like(sd["visual.trunk.patch_embed.proj.bias"])
    elif what == "q_bias_dropped":
        sd["visual.trunk.attn_pool.q.bias"] = torch.zeros_like(sd["visual.trunk.attn_pool.q.bias"])
    elif what == "pos_shifted":
        sd["visual.trunk.pos_embed"] = torch.roll(sd["visual.trunk.pos_embed"], 1, dims=1)
    return sd


@pytest.mark.timeout(600)
def test_bar_can_fail():
    """Two different inputs differ by 1 - cos >= 1e-2 in the oracle, and each wrong forward lands at least FLOOR times
    the bar away from the right one on at least one input of every case."""
    with torch.no_grad():
        for name, arch, sd in sensitivity_cases():
            px = structured_images(4, arch.image_size, 1)
            ids = captions(4, arch, 1)
            img = siglip_ref.image_features(sd, arch, px)
            txt = siglip_ref.text_features(sd, arch, ids)
            assert cos_dist(img[0], img[1]) >= 1e-2 and cos_dist(txt[0], txt[1]) >= 1e-2, name
            wrong_img = {
                "pool_no_residual": siglip_ref.image_features(sd, arch, px, wrong=("pool_no_residual",)),
                "kv_before_norm": siglip_ref.image_features(sd, arch, px, wrong=("kv_before_norm",)),
            }
            for what in ("patch_bias_dropped", "q_bias_dropped", "pos_shifted"):
                wrong_img[what] = siglip_ref.image_features(_mutated_sd(sd, what), arch, px)
            wrong_txt = {w: siglip_ref.text_features(sd, arch, ids, wrong=(w,)) for w in ("causal", "eot_pool")}
            for what, f in wrong_img.items():
                d = cos_dist(f, img).max()
                assert d >= FLOOR * COS_TOL, "%s / %s: 1 - cos %.2e" % (name, what, d)
            for what, f in wrong_txt.items():
                d = cos_dist(f, txt).max()
                assert d >= FLOOR * COS_TOL, "%s / %s: 1 - cos %.2e" % (name, what, d)
