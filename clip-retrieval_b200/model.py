"""The model object of the embed path and its loader.

Reference seam (SURVEY.md §8b B2): `all_clip.load_clip(clip_model, use_jit, warmup_batch_size,
clip_cache_path[, device]) -> (model, preprocess, tokenizer)` as called at
clip_retrieval/clip_inference/mapper.py:36-41, worker.py:52-57 and clip_back.py:868; the model is
used through `model.encode_image(Tensor[B,3,H,W]) -> Tensor[B,D]` and
`model.encode_text(Tensor[B,77]) -> Tensor[B,D]` (mapper.py:42-43,57,65; clip_back.py:230,244).
The forward runs in the CUDA library (include/b200clip.h, b200_clip_*); nothing here computes.
"""
import ctypes as C
import gzip
import html
import os
import threading
from dataclasses import dataclass
from functools import lru_cache

import numpy as np

from . import _lib
from ._lib import lib, check


@dataclass(frozen=True)
class Tower:
    width: int
    layers: int
    heads: int
    mlp: int


@dataclass(frozen=True)
class ClipArch:
    embed_dim: int
    image_size: int
    patch: int
    vision: Tower
    text: Tower
    context_length: int = 77
    vocab_size: int = 49408
    quick_gelu: bool = True


# Architectures the reference's docs and tests name (README.md:179,201,237; docs/laion5B_h14_back.md:60;
# tests/test_clip_inference/test_mapper.py:11-15).  Keys are the *architecture*; the activation follows the
# checkpoint family (OpenAI weights: QuickGELU; LAION open_clip weights: erf GELU) and is resolved by
# `resolve_arch` from the name's suffix / pretrained tag, as open_clip's factory does.
_B32 = (512, 224, 32, Tower(768, 12, 12, 3072), Tower(512, 12, 8, 2048))
_B16 = (512, 224, 16, Tower(768, 12, 12, 3072), Tower(512, 12, 8, 2048))
_L14 = (768, 224, 14, Tower(1024, 24, 16, 4096), Tower(768, 12, 12, 3072))
_L14_336 = (768, 336, 14, Tower(1024, 24, 16, 4096), Tower(768, 12, 12, 3072))
_H14 = (1024, 224, 14, Tower(1280, 32, 16, 5120), Tower(1024, 24, 16, 4096))
_B32_256 = (512, 256, 32, Tower(768, 12, 12, 3072), Tower(512, 12, 8, 2048))
# ViT-H/14 at 378 px (Apple's DFN5B weights, `ViT-H-14-378-quickgelu`): the H/14 towers with T = 27^2 + 1 = 730 image
# tokens.  Config recalled from open_clip's model config, not read from its source (DESIGN.md §5 (xvi)).
_H14_378 = (1024, 378, 14, Tower(1280, 32, 16, 5120), Tower(1024, 24, 16, 4096))

ARCHS = {
    # bare names -> OpenAI clip.load (QuickGELU)
    "ViT-B/32": ClipArch(*_B32, quick_gelu=True),
    "ViT-B/16": ClipArch(*_B16, quick_gelu=True),
    "ViT-L/14": ClipArch(*_L14, quick_gelu=True),
    "ViT-L/14@336px": ClipArch(*_L14_336, quick_gelu=True),
    # open_clip model configs (erf GELU unless `-quickgelu` / pretrained tag `openai`)
    "open_clip:ViT-B-32": ClipArch(*_B32, quick_gelu=False),
    "open_clip:ViT-B-32-256": ClipArch(*_B32_256, quick_gelu=False),
    "open_clip:ViT-B-16": ClipArch(*_B16, quick_gelu=False),
    "open_clip:ViT-L-14": ClipArch(*_L14, quick_gelu=False),
    "open_clip:ViT-L-14-336": ClipArch(*_L14_336, quick_gelu=False),
    "open_clip:ViT-H-14": ClipArch(*_H14, quick_gelu=False),
    "open_clip:ViT-H-14-378": ClipArch(*_H14_378, quick_gelu=False),
}
ARCHS["ViT-H/14"] = ARCHS["open_clip:ViT-H-14"]

# The two largest LAION CLIPs, whose image towers have head dims 88 (g) and 104 (bigG): 224 px, patch 14 (T = 257),
# context 77, erf GELU.  Configs recalled from open_clip's model configs (head_width 88 / 104, mlp_ratio 4.3637 / 4.9231
# -> int(width * ratio)) and the laion/CLIP-ViT-{g,bigG}-14 HuggingFace configs, not read from either (DESIGN.md §5
# (xvii)).  Kept apart from ARCHS, whose entries all have head dims in (64, 80, 96, 128); resolve_arch reads both.
_G14 = (1024, 224, 14, Tower(1408, 40, 16, 6144), Tower(1024, 24, 16, 4096))
_BIGG14 = (1280, 224, 14, Tower(1664, 48, 16, 8192), Tower(1280, 32, 20, 5120))
G14_ARCHS = {
    "open_clip:ViT-g-14": ClipArch(*_G14, quick_gelu=False),          # laion2b_s12b_b42k, laion2b_s34b_b88k
    "open_clip:ViT-bigG-14": ClipArch(*_BIGG14, quick_gelu=False),    # laion2b_s39b_b160k
}


@dataclass(frozen=True)
class ResNetArch:
    """OpenAI's ModifiedResNet image tower (include/b200clip.h b200_clip_create_resnet) with the CLIP text tower:
    `layers` Bottleneck blocks per stage, stem width `width` (stage i has planes width * 2^i), and an attention pool of
    32 * width channels in heads of 64."""
    embed_dim: int
    image_size: int
    layers: tuple
    width: int
    text: Tower
    context_length: int = 77
    vocab_size: int = 49408
    quick_gelu: bool = True

    @property
    def heads(self):
        return 32 * self.width // 64


# OpenAI's five ResNet CLIPs (clip.load names; open_clip serves the same towers as `open_clip:RN50[-quickgelu]/{openai,
# yfcc15m,cc12m}`, `open_clip:RN101[-quickgelu]/{openai,yfcc15m}`, `open_clip:RN50x{4,16,64}/openai`).  Configs recalled
# from OpenAI's and open_clip's model configs, not read from either (DESIGN.md §5 (xviii)).  Kept apart from ARCHS and
# G14_ARCHS, whose entries are ViTs; resolve_arch reads all three.
_RN = {
    "RN50": (1024, 224, (3, 4, 6, 3), 64, Tower(512, 12, 8, 2048)),
    "RN101": (512, 224, (3, 4, 23, 3), 64, Tower(512, 12, 8, 2048)),
    "RN50x4": (640, 288, (4, 6, 10, 6), 80, Tower(640, 12, 10, 2560)),
    "RN50x16": (768, 384, (6, 8, 18, 8), 96, Tower(768, 12, 12, 3072)),
    "RN50x64": (1024, 448, (3, 15, 36, 10), 128, Tower(1024, 12, 16, 4096)),
}
RESNET_ARCHS = {}
for _k, _a in _RN.items():
    RESNET_ARCHS[_k] = ResNetArch(*_a, quick_gelu=True)                   # bare names -> OpenAI clip.load
    RESNET_ARCHS["open_clip:" + _k] = ResNetArch(*_a, quick_gelu=False)   # QuickGELU with `-quickgelu` / `openai`


@dataclass(frozen=True)
class SigLIPArch:
    """Google's SigLIP as open_clip builds it (include/b200clip.h b200_clip_create_siglip): a timm ViT image tower with
    a latent-query attention pool and no projection (embed_dim == vision.width), and a bidirectional text tower pooled
    at its last position with a biased projection.  LayerNorm eps 1e-6 and erf GELU throughout.  `tokenizer` names
    the HuggingFace repository folder whose tokenizer.json the model uses."""
    embed_dim: int
    image_size: int
    patch: int
    vision: Tower
    text: Tower
    context_length: int = 64
    vocab_size: int = 32000
    tokenizer: str = "timm/ViT-B-16-SigLIP"
    quick_gelu: bool = False


# open_clip's SigLIP configs (pretrained tag `webli`), recalled from open_clip's model configs, not read
# (DESIGN.md §5 (xix)).  Kept apart from ARCHS, G14_ARCHS and RESNET_ARCHS; resolve_arch reads all four.
_SIG_B = Tower(768, 12, 12, 3072)
_SIG_L = Tower(1024, 24, 16, 4096)
_SIG_SO = Tower(1152, 27, 16, 4304)
SIGLIP_ARCHS = {
    "open_clip:ViT-B-16-SigLIP": SigLIPArch(768, 224, 16, _SIG_B, _SIG_B),
    "open_clip:ViT-B-16-SigLIP-256": SigLIPArch(768, 256, 16, _SIG_B, _SIG_B),
    "open_clip:ViT-B-16-SigLIP-384": SigLIPArch(768, 384, 16, _SIG_B, _SIG_B),
    "open_clip:ViT-B-16-SigLIP-512": SigLIPArch(768, 512, 16, _SIG_B, _SIG_B),
    "open_clip:ViT-B-16-SigLIP-i18n-256": SigLIPArch(768, 256, 16, _SIG_B, _SIG_B, vocab_size=250000,
                                                     tokenizer="timm/ViT-B-16-SigLIP-i18n-256"),
    "open_clip:ViT-L-16-SigLIP-256": SigLIPArch(1024, 256, 16, _SIG_L, _SIG_L),
    "open_clip:ViT-L-16-SigLIP-384": SigLIPArch(1024, 384, 16, _SIG_L, _SIG_L),
    "open_clip:ViT-SO400M-14-SigLIP": SigLIPArch(1152, 224, 14, _SIG_SO, _SIG_SO, context_length=16),
    "open_clip:ViT-SO400M-14-SigLIP-384": SigLIPArch(1152, 384, 14, _SIG_SO, _SIG_SO),
}


@dataclass(frozen=True)
class ConvNeXtArch:
    """open_clip's ConvNeXt CLIPs (include/b200clip.h b200_clip_create_convnext): timm's ConvNeXt trunk (`depths` blocks
    per stage at widths `dims`, every LayerNorm at `eps`) under open_clip's linear or MLP (`head_mlp`) head, with the
    standard CLIP text tower (erf GELU).  `tags` are the pretrained tags open_clip publishes for the name."""
    embed_dim: int
    image_size: int
    depths: tuple
    dims: tuple
    head_mlp: bool
    text: Tower
    eps: float = 1e-6
    tags: tuple = ()
    context_length: int = 77
    vocab_size: int = 49408
    quick_gelu: bool = False


# open_clip's ConvNeXt configs and pretrained tags, recalled from open_clip's model and pretrained configs and timm's
# ConvNeXt, not read from any of them (DESIGN.md §5 (xx)); xxlarge's LayerNorm eps 1e-5 is timm's `norm_eps` for it.
# Kept apart from ARCHS, G14_ARCHS, RESNET_ARCHS and SIGLIP_ARCHS; resolve_arch reads all five.
_CNX_BASE = ((3, 3, 27, 3), (128, 256, 512, 1024))
_CNX_LARGE = ((3, 3, 27, 3), (192, 384, 768, 1536))
_CNX_XXL = ((3, 4, 30, 3), (384, 768, 1536, 3072))
CONVNEXT_ARCHS = {
    "open_clip:convnext_base": ConvNeXtArch(512, 224, *_CNX_BASE, False, Tower(512, 12, 8, 2048),
                                            tags=("laion400m_s13b_b51k",)),
    "open_clip:convnext_base_w": ConvNeXtArch(640, 256, *_CNX_BASE, False, Tower(640, 12, 10, 2560),
                                              tags=("laion2b_s13b_b82k", "laion2b_s13b_b82k_augreg",
                                                    "laion_aesthetic_s13b_b82k")),
    "open_clip:convnext_base_w_320": ConvNeXtArch(640, 320, *_CNX_BASE, False, Tower(640, 12, 10, 2560),
                                                  tags=("laion_aesthetic_s13b_b82k", "laion_aesthetic_s13b_b82k_augreg")),
    "open_clip:convnext_large_d": ConvNeXtArch(768, 256, *_CNX_LARGE, True, Tower(768, 16, 12, 3072),
                                               tags=("laion2b_s26b_b102k_augreg",)),
    "open_clip:convnext_large_d_320": ConvNeXtArch(768, 320, *_CNX_LARGE, True, Tower(768, 16, 12, 3072),
                                                   tags=("laion2b_s29b_b131k_ft", "laion2b_s29b_b131k_ft_soup")),
    "open_clip:convnext_xxlarge": ConvNeXtArch(1024, 256, *_CNX_XXL, False, Tower(1024, 24, 16, 4096), eps=1e-5,
                                               tags=("laion2b_s34b_b82k_augreg", "laion2b_s34b_b82k_augreg_rewind",
                                                     "laion2b_s34b_b82k_augreg_soup")),
}

# Every architecture a `clip_model` name can resolve to.
KNOWN_ARCHS = {**ARCHS, **G14_ARCHS, **RESNET_ARCHS, **SIGLIP_ARCHS, **CONVNEXT_ARCHS}

# `hf_clip:<repo>` names -> (architecture key, quick_gelu): HuggingFace CLIPModel checkpoints of the same towers.
HF_REPOS = {
    "openai/clip-vit-base-patch32": ("open_clip:ViT-B-32", True),
    "openai/clip-vit-base-patch16": ("open_clip:ViT-B-16", True),
    "openai/clip-vit-large-patch14": ("open_clip:ViT-L-14", True),
    "openai/clip-vit-large-patch14-336": ("open_clip:ViT-L-14-336", True),
    "patrickjohncyh/fashion-clip": ("open_clip:ViT-B-32", True),      # fine-tuned from openai/clip-vit-base-patch32
    "laion/CLIP-ViT-B-32-laion2B-s34B-b79K": ("open_clip:ViT-B-32", False),
    "laion/CLIP-ViT-L-14-laion2B-s32B-b82K": ("open_clip:ViT-L-14", False),
    "laion/CLIP-ViT-H-14-laion2B-s32B-b79K": ("open_clip:ViT-H-14", False),
    "laion/CLIP-ViT-g-14-laion2B-s12B-b42K": ("open_clip:ViT-g-14", False),
    "laion/CLIP-ViT-g-14-laion2B-s34B-b88K": ("open_clip:ViT-g-14", False),
    "laion/CLIP-ViT-bigG-14-laion2B-39B-b160k": ("open_clip:ViT-bigG-14", False),
}
# `nm:<repo>` (DeepSparse, README.md:201) names quantised ONNX exports of these open_clip towers.
NM_REPOS = {
    "neuralmagic/CLIP-ViT-B-32-256x256-DataComp-s34B-b86K-quant-ds": ("open_clip:ViT-B-32-256", False),
    "mgoin/CLIP-ViT-B-32-laion2b_s34b_b79k-ds": ("open_clip:ViT-B-32", False),
}


def _torch():
    import torch

    return torch


def arch_from_hf_config(cfg):
    """ClipArch from a HuggingFace CLIPConfig dict (config.json of an `hf_clip:` repo)."""
    v, t = cfg["vision_config"], cfg["text_config"]
    act = v.get("hidden_act", "quick_gelu")
    if act not in ("quick_gelu", "gelu"):
        raise ValueError("hf_clip: activation %r not supported" % act)
    return ClipArch(int(cfg.get("projection_dim", v.get("projection_dim", 512))), int(v.get("image_size", 224)),
                    int(v.get("patch_size", 32)),
                    Tower(int(v["hidden_size"]), int(v["num_hidden_layers"]), int(v["num_attention_heads"]), int(v["intermediate_size"])),
                    Tower(int(t["hidden_size"]), int(t["num_hidden_layers"]), int(t["num_attention_heads"]), int(t["intermediate_size"])),
                    int(t.get("max_position_embeddings", 77)), int(t.get("vocab_size", 49408)), quick_gelu=(act == "quick_gelu"))


def resolve_arch(clip_model):
    """Map a reference `clip_model` string to (arch, key) the way all_clip's dispatcher reads it
    (README.md:179,201,237): bare names are OpenAI checkpoints (QuickGELU); `open_clip:ARCH[/PRETRAINED]`
    is an open_clip model config, QuickGELU when ARCH ends in `-quickgelu` or PRETRAINED is `openai`
    (open_clip's factory forces it for OpenAI weights); `hf_clip:REPO` / `nm:REPO` name a known repo."""
    from dataclasses import replace

    name = clip_model
    if name.startswith("synthetic:"):
        name = name[len("synthetic:"):]
    if name.startswith("open_clip:"):
        spec = name[len("open_clip:"):]
        arch_name, _, pretrained = spec.partition("/")
        quick = False
        if arch_name.endswith("-quickgelu"):
            arch_name, quick = arch_name[: -len("-quickgelu")], True
        if pretrained == "openai":
            quick = True
        key = "open_clip:" + arch_name
        if key in SIGLIP_ARCHS:
            if quick or pretrained not in ("", "webli"):
                raise ValueError("%r: SigLIP models take erf GELU and the `webli` weights only (no -quickgelu, no "
                                 "`openai` tag)" % (clip_model,))
            return SIGLIP_ARCHS[key], key
        if key in CONVNEXT_ARCHS:
            arch = CONVNEXT_ARCHS[key]
            if quick:
                raise ValueError("%r: the ConvNeXt CLIPs take erf GELU and LAION weights only (no -quickgelu, no "
                                 "`openai` tag)" % (clip_model,))
            if pretrained and pretrained not in arch.tags:
                raise ValueError("%r: unknown pretrained tag; %s has %s" % (clip_model, arch_name, ", ".join(arch.tags)))
            # the tag stays in the key: checkpoints are looked up as `<name>-<tag>.pt`
            return arch, key + ("/" + pretrained if pretrained else "")
        if key not in KNOWN_ARCHS:
            raise ValueError("unknown clip_model %r; known: %s" % (clip_model, ", ".join(sorted(KNOWN_ARCHS))))
        return replace(KNOWN_ARCHS[key], quick_gelu=quick), key + ("-quickgelu" if quick else "")
    for prefix, table in (("hf_clip:", HF_REPOS), ("nm:", NM_REPOS)):
        if name.startswith(prefix):
            repo = name[len(prefix):]
            if repo not in table:
                raise ValueError("unknown %s repository %r; known: %s (or load a state_dict with "
                                 "B200Clip(arch_from_hf_config(config)))" % (prefix, repo, ", ".join(sorted(table))))
            key, quick = table[repo]
            return replace(KNOWN_ARCHS[key], quick_gelu=quick), name
    if name not in KNOWN_ARCHS:
        raise ValueError("unknown clip_model %r; known: %s" % (clip_model, ", ".join(sorted(KNOWN_ARCHS))))
    return KNOWN_ARCHS[name], name


def synthetic_state_dict(arch, seed=0):
    """Seeded random-init weights in the OpenAI/open_clip key layout (benchmarks run on random
    weights of the named architecture: there is no network for checkpoints)."""
    torch = _torch()
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    sd = {}
    if isinstance(arch, SigLIPArch):
        return _siglip_state_dict(arch, rn)
    if isinstance(arch, ResNetArch):
        _resnet_visual(sd, arch, rn, g)
    if isinstance(arch, ConvNeXtArch):
        _convnext_visual(sd, arch, rn, g)

    def tower(prefix, t):
        w, L = t.width, t.layers
        for i in range(L):
            p = "%stransformer.resblocks.%d." % (prefix, i)
            sd[p + "ln_1.weight"] = 1.0 + rn(w, std=0.1)
            sd[p + "ln_1.bias"] = rn(w, std=0.05)
            sd[p + "attn.in_proj_weight"] = rn(3 * w, w, std=w ** -0.5)
            sd[p + "attn.in_proj_bias"] = rn(3 * w, std=0.02)
            sd[p + "attn.out_proj.weight"] = rn(w, w, std=(w ** -0.5) * ((2 * L) ** -0.5))
            sd[p + "attn.out_proj.bias"] = rn(w, std=0.02)
            sd[p + "ln_2.weight"] = 1.0 + rn(w, std=0.1)
            sd[p + "ln_2.bias"] = rn(w, std=0.05)
            sd[p + "mlp.c_fc.weight"] = rn(t.mlp, w, std=(2 * w) ** -0.5)
            sd[p + "mlp.c_fc.bias"] = rn(t.mlp, std=0.02)
            sd[p + "mlp.c_proj.weight"] = rn(w, t.mlp, std=(w ** -0.5) * ((2 * L) ** -0.5))
            sd[p + "mlp.c_proj.bias"] = rn(w, std=0.02)

    t = arch.text
    if not isinstance(arch, (ResNetArch, ConvNeXtArch)):
        v = arch.vision
        grid = arch.image_size // arch.patch
        sd["visual.conv1.weight"] = rn(v.width, 3, arch.patch, arch.patch, std=(3 * arch.patch ** 2) ** -0.5)
        sd["visual.class_embedding"] = rn(v.width, std=v.width ** -0.5)
        sd["visual.positional_embedding"] = rn(grid * grid + 1, v.width, std=v.width ** -0.5)
        sd["visual.ln_pre.weight"] = 1.0 + rn(v.width, std=0.1)
        sd["visual.ln_pre.bias"] = rn(v.width, std=0.05)
        tower("visual.", v)
        sd["visual.ln_post.weight"] = 1.0 + rn(v.width, std=0.1)
        sd["visual.ln_post.bias"] = rn(v.width, std=0.05)
        sd["visual.proj"] = rn(v.width, arch.embed_dim, std=v.width ** -0.5)
    sd["token_embedding.weight"] = rn(arch.vocab_size, t.width, std=0.02)
    sd["positional_embedding"] = rn(arch.context_length, t.width, std=0.01)
    tower("", t)
    sd["ln_final.weight"] = 1.0 + rn(t.width, std=0.1)
    sd["ln_final.bias"] = rn(t.width, std=0.05)
    sd["text_projection"] = rn(t.width, arch.embed_dim, std=t.width ** -0.5)
    return sd


def _siglip_state_dict(arch, rn):
    """SigLIP weights in open_clip's layout (visual.trunk.* from timm, text.*), with non-trivial LayerNorm affines
    and biases."""
    sd = {}

    def ln(name, n):
        sd[name + ".weight"] = 1.0 + rn(n, std=0.1)
        sd[name + ".bias"] = rn(n, std=0.05)

    def linear(name, n_out, n_in, std):
        sd[name + ".weight"] = rn(n_out, n_in, std=std)
        sd[name + ".bias"] = rn(n_out, std=0.02)

    def mlp(prefix, a, b, w, h, L):
        linear(prefix + a, h, w, (2 * w) ** -0.5)
        linear(prefix + b, w, h, (w ** -0.5) * ((2 * L) ** -0.5))

    v, t, p = arch.vision, arch.text, arch.patch
    w, L, grid = v.width, v.layers, arch.image_size // p
    tr = "visual.trunk."
    linear(tr + "patch_embed.proj", w, 3 * p * p, (3 * p * p) ** -0.5)
    sd[tr + "patch_embed.proj.weight"] = sd[tr + "patch_embed.proj.weight"].reshape(w, 3, p, p)
    sd[tr + "pos_embed"] = rn(1, grid * grid, w, std=w ** -0.5)
    for i in range(L):
        b = "%sblocks.%d." % (tr, i)
        ln(b + "norm1", w)
        linear(b + "attn.qkv", 3 * w, w, w ** -0.5)
        linear(b + "attn.proj", w, w, (w ** -0.5) * ((2 * L) ** -0.5))
        ln(b + "norm2", w)
        mlp(b, "mlp.fc1", "mlp.fc2", w, v.mlp, L)
    ln(tr + "norm", w)
    a = tr + "attn_pool."
    sd[a + "latent"] = rn(1, 1, w, std=w ** -0.5)
    linear(a + "q", w, w, w ** -0.5)
    linear(a + "kv", 2 * w, w, w ** -0.5)
    linear(a + "proj", w, w, w ** -0.5)
    ln(a + "norm", w)
    mlp(a, "mlp.fc1", "mlp.fc2", w, v.mlp, 1)
    tw, tL = t.width, t.layers
    sd["text.token_embedding.weight"] = rn(arch.vocab_size, tw, std=0.02)
    sd["text.positional_embedding"] = rn(arch.context_length, tw, std=0.01)
    for i in range(tL):
        q = "text.transformer.resblocks.%d." % i
        ln(q + "ln_1", tw)
        sd[q + "attn.in_proj_weight"] = rn(3 * tw, tw, std=tw ** -0.5)
        sd[q + "attn.in_proj_bias"] = rn(3 * tw, std=0.02)
        linear(q + "attn.out_proj", tw, tw, (tw ** -0.5) * ((2 * tL) ** -0.5))
        ln(q + "ln_2", tw)
        mlp(q, "mlp.c_fc", "mlp.c_proj", tw, t.mlp, tL)
    ln("text.ln_final", tw)
    linear("text.text_projection", arch.embed_dim, tw, tw ** -0.5)
    return sd


def _resnet_visual(sd, arch, rn, g):
    """visual.* of a ResNetArch in OpenAI's key layout: He-scaled convolutions, and BatchNorm layers with non-trivial
    affine and running statistics (so a forward that skips or misplaces the fold is visibly wrong).  bn3 of each block
    is scaled down (OpenAI zero-initialises it) so that the residual stream stays O(1) at depth."""
    torch = _torch()
    w = arch.width

    def conv(name, cout, cin, k):
        sd[name + ".weight"] = rn(cout, cin, k, k, std=(2.0 / (cin * k * k)) ** 0.5)

    def bn(name, n, gain=1.0):
        sd[name + ".weight"] = gain * (1.0 + rn(n, std=0.2))
        sd[name + ".bias"] = rn(n, std=0.1)
        sd[name + ".running_mean"] = rn(n, std=0.2)
        sd[name + ".running_var"] = 0.5 + torch.rand(n, generator=g)
        sd[name + ".num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)

    conv("visual.conv1", w // 2, 3, 3)
    bn("visual.bn1", w // 2)
    conv("visual.conv2", w // 2, w // 2, 3)
    bn("visual.bn2", w // 2)
    conv("visual.conv3", w, w // 2, 3)
    bn("visual.bn3", w)
    cin = w
    for s, n in enumerate(arch.layers):
        planes = w << s
        for j in range(n):
            p = "visual.layer%d.%d." % (s + 1, j)
            conv(p + "conv1", planes, cin, 1)
            bn(p + "bn1", planes)
            conv(p + "conv2", planes, planes, 3)
            bn(p + "bn2", planes)
            conv(p + "conv3", 4 * planes, planes, 1)
            bn(p + "bn3", 4 * planes, gain=0.3)
            if (j == 0 and s > 0) or cin != 4 * planes:
                conv(p + "downsample.0", 4 * planes, cin, 1)
                bn(p + "downsample.1", 4 * planes)
            cin = 4 * planes
    C, T = 32 * w, (arch.image_size // 32) ** 2 + 1
    a = "visual.attnpool."
    sd[a + "positional_embedding"] = rn(T, C, std=C ** -0.5)
    for n in ("q", "k", "v"):
        sd[a + n + "_proj.weight"] = rn(C, C, std=C ** -0.5)
        sd[a + n + "_proj.bias"] = rn(C, std=0.02)
    sd[a + "c_proj.weight"] = rn(arch.embed_dim, C, std=C ** -0.5)
    sd[a + "c_proj.bias"] = rn(arch.embed_dim, std=0.02)


def _convnext_visual(sd, arch, rn, g):
    """visual.trunk.* and visual.head.* of a ConvNeXtArch in open_clip's layout, with non-trivial LayerNorm affines and
    biases and layer scales gamma uniform in [0.1, 1] (real checkpoints start them at 1e-6; near zero, every block
    would vanish from the output and a wrong block would go unseen)."""
    torch = _torch()
    t = "visual.trunk."

    def ln(name, n):
        sd[name + ".weight"] = 1.0 + rn(n, std=0.1)
        sd[name + ".bias"] = rn(n, std=0.05)

    def lin(name, n_out, n_in, bias=True):
        sd[name + ".weight"] = rn(n_out, n_in, std=n_in ** -0.5)
        if bias:
            sd[name + ".bias"] = rn(n_out, std=0.02)

    C0 = arch.dims[0]
    sd[t + "stem.0.weight"] = rn(C0, 3, 4, 4, std=48 ** -0.5)
    sd[t + "stem.0.bias"] = rn(C0, std=0.02)
    ln(t + "stem.1", C0)
    for s, (n, C) in enumerate(zip(arch.depths, arch.dims)):
        p = "%sstages.%d." % (t, s)
        if s > 0:
            Cp = arch.dims[s - 1]
            ln(p + "downsample.0", Cp)
            sd[p + "downsample.1.weight"] = rn(C, Cp, 2, 2, std=(4 * Cp) ** -0.5)
            sd[p + "downsample.1.bias"] = rn(C, std=0.02)
        for j in range(n):
            b = "%sblocks.%d." % (p, j)
            sd[b + "conv_dw.weight"] = rn(C, 1, 7, 7, std=49 ** -0.5)
            sd[b + "conv_dw.bias"] = rn(C, std=0.05)
            ln(b + "norm", C)
            lin(b + "mlp.fc1", 4 * C, C)
            lin(b + "mlp.fc2", C, 4 * C)
            sd[b + "gamma"] = 0.1 + 0.9 * torch.rand(C, generator=g)
    C3, D = arch.dims[3], arch.embed_dim
    ln(t + "head.norm", C3)
    if arch.head_mlp:
        lin("visual.head.mlp.fc1", 2 * D, C3)
        lin("visual.head.mlp.fc2", D, 2 * D, bias=False)
    else:
        lin("visual.head.proj", D, C3, bias=False)


def convert_hf_state_dict(sd, arch):
    """HuggingFace CLIPModel parameter names (`hf_clip:` models) -> the OpenAI/open_clip layout."""
    torch = _torch()
    out = {}

    def tower(src, dst, t):
        for i in range(t.layers):
            s = "%sencoder.layers.%d." % (src, i)
            d = "%stransformer.resblocks.%d." % (dst, i)
            out[d + "attn.in_proj_weight"] = torch.cat([sd[s + "self_attn.%s_proj.weight" % n] for n in "qkv"], 0)
            out[d + "attn.in_proj_bias"] = torch.cat([sd[s + "self_attn.%s_proj.bias" % n] for n in "qkv"], 0)
            out[d + "attn.out_proj.weight"] = sd[s + "self_attn.out_proj.weight"]
            out[d + "attn.out_proj.bias"] = sd[s + "self_attn.out_proj.bias"]
            for a, b in (("ln_1", "layer_norm1"), ("ln_2", "layer_norm2")):
                out[d + a + ".weight"], out[d + a + ".bias"] = sd[s + b + ".weight"], sd[s + b + ".bias"]
            for a, b in (("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
                out[d + a + ".weight"], out[d + a + ".bias"] = sd[s + b + ".weight"], sd[s + b + ".bias"]

    tower("vision_model.", "visual.", arch.vision)
    tower("text_model.", "", arch.text)
    out["visual.conv1.weight"] = sd["vision_model.embeddings.patch_embedding.weight"]
    out["visual.class_embedding"] = sd["vision_model.embeddings.class_embedding"]
    out["visual.positional_embedding"] = sd["vision_model.embeddings.position_embedding.weight"]
    out["visual.ln_pre.weight"], out["visual.ln_pre.bias"] = sd["vision_model.pre_layrnorm.weight"], sd["vision_model.pre_layrnorm.bias"]
    out["visual.ln_post.weight"], out["visual.ln_post.bias"] = sd["vision_model.post_layernorm.weight"], sd["vision_model.post_layernorm.bias"]
    out["visual.proj"] = sd["visual_projection.weight"].t().contiguous()
    out["token_embedding.weight"] = sd["text_model.embeddings.token_embedding.weight"]
    out["positional_embedding"] = sd["text_model.embeddings.position_embedding.weight"]
    out["ln_final.weight"], out["ln_final.bias"] = sd["text_model.final_layer_norm.weight"], sd["text_model.final_layer_norm.bias"]
    out["text_projection"] = sd["text_projection.weight"].t().contiguous()
    return out


class B200Clip:
    """CLIP towers on one GPU.  `encode_image` / `encode_text` follow the reference model's
    contract (CUDA tensors in, fp32 feature tensor out); `embed_*` fuse the normalise + cast of
    mapper.py:58-59,66-67 into the last kernel and are what `ClipMapper` calls."""

    def __init__(self, arch, device=0, max_batch=256):
        self.arch = arch
        self.device_index = int(device)
        self.max_batch = int(max_batch)
        self._h = C.c_void_p()
        self._lock = threading.Lock()
        if isinstance(arch, SigLIPArch):
            cfg = _lib.ClipConfigC(
                arch.embed_dim, arch.image_size, arch.patch,
                _lib.TowerConfigC(arch.vision.width, arch.vision.layers, arch.vision.heads, arch.vision.mlp),
                arch.context_length, arch.vocab_size,
                _lib.TowerConfigC(arch.text.width, arch.text.layers, arch.text.heads, arch.text.mlp),
                0, self.max_batch,
            )
            check(lib.b200_clip_create_siglip(C.byref(cfg), self.device_index, C.byref(self._h)), "clip_create_siglip")
            return
        if isinstance(arch, ConvNeXtArch):
            cfg = _lib.ClipConfigC(
                arch.embed_dim, arch.image_size, 0, _lib.TowerConfigC(0, 0, 0, 0), arch.context_length, arch.vocab_size,
                _lib.TowerConfigC(arch.text.width, arch.text.layers, arch.text.heads, arch.text.mlp),
                1 if arch.quick_gelu else 0, self.max_batch,
            )
            nc = _lib.ConvNeXtConfigC((C.c_int32 * 4)(*arch.depths), (C.c_int32 * 4)(*arch.dims),
                                      1 if arch.head_mlp else 0, arch.eps)
            check(lib.b200_clip_create_convnext(C.byref(cfg), C.byref(nc), self.device_index, C.byref(self._h)),
                  "clip_create_convnext")
            return
        if isinstance(arch, ResNetArch):
            cfg = _lib.ClipConfigC(
                arch.embed_dim, arch.image_size, 0, _lib.TowerConfigC(0, 0, 0, 0), arch.context_length, arch.vocab_size,
                _lib.TowerConfigC(arch.text.width, arch.text.layers, arch.text.heads, arch.text.mlp),
                1 if arch.quick_gelu else 0, self.max_batch,
            )
            rc = _lib.ResNetConfigC((C.c_int32 * 4)(*arch.layers), arch.width, arch.heads)
            check(lib.b200_clip_create_resnet(C.byref(cfg), C.byref(rc), self.device_index, C.byref(self._h)),
                  "clip_create_resnet")
            return
        cfg = _lib.ClipConfigC(
            arch.embed_dim, arch.image_size, arch.patch,
            _lib.TowerConfigC(arch.vision.width, arch.vision.layers, arch.vision.heads, arch.vision.mlp),
            arch.context_length, arch.vocab_size,
            _lib.TowerConfigC(arch.text.width, arch.text.layers, arch.text.heads, arch.text.mlp),
            1 if arch.quick_gelu else 0, self.max_batch,
        )
        check(lib.b200_clip_create(C.byref(cfg), self.device_index, C.byref(self._h)), "clip_create")

    def __del__(self):
        try:
            if self._h:
                lib.b200_clip_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    # ---- weights ----
    def load_state_dict(self, sd):
        """sd: name -> torch tensor / numpy array (fp32 or fp16), OpenAI/open_clip key layout."""
        views, keep = _tensor_views(sd)
        check(lib.b200_clip_load_weights(self._h, views, len(keep)), "clip_load_weights")
        return self

    # ---- reference model contract ----
    @property
    def device(self):
        return _torch().device("cuda", self.device_index)

    def _encode_device(self, x, image, out_dtype, normalize):
        torch = _torch()
        if not x.is_cuda:
            x = x.to(self.device)
        if image:
            s = self.arch.image_size
            if x.dim() != 4 or tuple(x.shape[1:]) != (3, s, s):
                raise ValueError("encode_image: expected [B,3,%d,%d], got %r" % (s, s, tuple(x.shape)))
            x = x.to(torch.float32).contiguous()
        else:
            if x.dim() != 2 or x.shape[1] != self.arch.context_length:
                raise ValueError("encode_text: expected [B,%d], got %r" % (self.arch.context_length, tuple(x.shape)))
            x = x.to(torch.int64).contiguous()
        B = x.shape[0]
        out = torch.empty((B, self.arch.embed_dim), dtype=out_dtype, device=x.device)
        code = 1 if out_dtype == torch.float16 else 0
        st = torch.cuda.current_stream(x.device).cuda_stream
        fn = lib.b200_clip_encode_image_device if image else lib.b200_clip_encode_text_device
        with self._lock:  # one forward at a time per handle (clip_back serves from Flask threads)
            check(fn(self._h, x.data_ptr(), B, out.data_ptr(), code, 1 if normalize else 0, st), "clip_encode")
        return out

    def encode_image(self, image):
        return self._encode_device(image, True, _torch().float32, False)

    def encode_text(self, text):
        return self._encode_device(text, False, _torch().float32, False)

    # ---- fused mapper path ----
    def embed_image_device(self, image, dtype=None, normalize=True):
        return self._encode_device(image, True, dtype or _torch().float16, normalize)

    def embed_text_device(self, text, dtype=None, normalize=True):
        return self._encode_device(text, False, dtype or _torch().float16, normalize)

    def _embed_host(self, x, image, np_dtype):
        """Host tensor / array in, numpy out: H2D, forward, D2H inside one library call."""
        if _is_torch(x):
            torch = _torch()
            x = x.detach()
            if x.is_cuda:
                out = self._encode_device(x, image, torch.float16 if np_dtype == np.float16 else torch.float32, True)
                return out.cpu().numpy()
            x = x.to(torch.float32 if image else torch.int64).contiguous().numpy()
        else:
            x = np.ascontiguousarray(x, dtype=np.float32 if image else np.int64)
        if not image and isinstance(self.arch, SigLIPArch) and (x.ndim != 2 or x.shape[1] != self.arch.context_length):
            # the pads take part in SigLIP's attention and position T - 1 is pooled: no other width means the same
            raise ValueError("embed_text: expected token ids [B, %d], got %r" % (self.arch.context_length, x.shape))
        B = x.shape[0]
        out = np.empty((B, self.arch.embed_dim), dtype=np_dtype)
        fn = lib.b200_clip_encode_image if image else lib.b200_clip_encode_text
        check(fn(self._h, x.ctypes.data, B, out.ctypes.data, 1 if np_dtype == np.float16 else 0, 1), "clip_encode")
        return out

    def embed_image(self, image_tensor):
        """mapper.py:57-59 in one call: np.float16 [B, D], L2-normalised."""
        return self._embed_host(image_tensor, True, np.float16)

    def embed_text(self, text_tokens):
        """mapper.py:65-67 in one call."""
        return self._embed_host(text_tokens, False, np.float16)

    def set_profiling(self, on):
        check(lib.b200_clip_set_profiling(self._h, 1 if on else 0), "set_profiling")

    def last_timing(self):
        ms = (C.c_float * 8)()
        n = C.c_int(0)
        check(lib.b200_clip_last_timing(self._h, ms, C.byref(n)), "last_timing")
        return {"gemm": ms[0], "attention": ms[1], "layernorm": ms[2], "other": ms[3], "launches": int(n.value),
                "gemm_by_kind": {"qkv": ms[4], "out_proj": ms[5], "fc": ms[6], "c_proj": ms[7]}}


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _tensor_views(sd):
    """b200_tensor_view array over a state_dict (fp32 / fp16 host copies; tensors of more than 4 dimensions are
    skipped) and the arrays it points into, which the caller keeps alive for the duration of the call."""
    torch = _torch()
    views = (_lib.TensorViewC * len(sd))()
    keep = []
    for name, t in sd.items():
        if _is_torch(t):
            t = t.detach().cpu()
            if t.dtype not in (torch.float32, torch.float16):
                t = t.float()
            a = t.contiguous().numpy()
        else:
            a = np.ascontiguousarray(t)
            if a.dtype not in (np.float32, np.float16):
                a = a.astype(np.float32)
        if a.ndim > 4:
            continue
        v = views[len(keep)]
        keep.append(a)
        v.name = name.encode()
        v.data = a.ctypes.data
        v.dtype = 0 if a.dtype == np.float32 else 1
        v.ndim = a.ndim
        for i, s in enumerate(a.shape):
            v.shape[i] = s
    return views, keep


# ---- preprocess / tokenizer (returned by load_clip for signature parity; reader-side, CPU) ----------

# open_clip pretrained tags whose transform squashes the image to n_px x n_px instead of resizing the shorter side
# and cropping (resize_mode="squash" in open_clip's pretrained config, as recalled: DESIGN.md §5 (xvi)).
_SQUASH_TAGS = {"open_clip:ViT-H-14-378": ("dfn5b",)}


OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
# SigLIP's transform (open_clip's pretrained config for every `webli` SigLIP, as recalled: DESIGN.md §5 (xix)): squash
# to n_px x n_px, bicubic, and normalise with mean = std = 0.5.
SIGLIP_MEAN = SIGLIP_STD = (0.5, 0.5, 0.5)


def preprocess_mode(clip_model):
    """"squash" or "shortest": the resize step of the transform `load_clip` returns for this name (and that
    `ClipMapper` runs on the GPU for `image_rgb8` batches)."""
    return preprocess_params(clip_model)[0]


def preprocess_params(clip_model):
    """(resize mode, mean, std) of the transform `load_clip` returns for this name, and that `ClipMapper` runs on the
    GPU for `image_rgb8` batches."""
    name = clip_model[len("synthetic:"):] if clip_model.startswith("synthetic:") else clip_model
    if name.startswith("open_clip:"):
        arch_name, _, pretrained = name.partition("/")
        if arch_name in SIGLIP_ARCHS:
            return "squash", SIGLIP_MEAN, SIGLIP_STD
        if arch_name.endswith("-quickgelu"):
            arch_name = arch_name[: -len("-quickgelu")]
        if pretrained in _SQUASH_TAGS.get(arch_name, ()):
            return "squash", OPENAI_MEAN, OPENAI_STD
    return "shortest", OPENAI_MEAN, OPENAI_STD


def make_preprocess(n_px, resize_mode="shortest", mean=OPENAI_MEAN, std=OPENAI_STD):
    """torchvision Compose[Resize(n_px, BICUBIC), CenterCrop, RGB, ToTensor, Normalize(mean, std)] (OpenAI's mean /
    std by default) — the transform SURVEY.md §4 verified bit-exactly against the reference's test_tensors fixtures.
    With resize_mode "squash", Resize((n_px, n_px), BICUBIC) and no crop."""
    from torchvision import transforms as T
    from torchvision.transforms import InterpolationMode

    if resize_mode not in ("shortest", "squash"):
        raise ValueError("resize_mode %r: 'shortest' or 'squash'" % (resize_mode,))
    size = (n_px, n_px) if resize_mode == "squash" else n_px
    return T.Compose([
        T.Resize(size, interpolation=InterpolationMode.BICUBIC),
        T.CenterCrop(n_px),
        lambda im: im.convert("RGB"),
        T.ToTensor(),
        T.Normalize(mean, std),
    ])


class SimpleTokenizer:
    """CLIP byte-pair tokenizer over `bpe_simple_vocab_16e6.txt.gz` (shipped by clip/open_clip, not
    present offline).  Callable: tokenizer(list[str]) -> LongTensor [n, 77] with SOT 49406, EOT
    49407, zero padding, truncation keeping EOT last (reference HISTORY.md:47-49)."""

    def __init__(self, bpe_path, context_length=77):
        self.context_length = context_length
        merges = gzip.open(bpe_path).read().decode("utf-8").split("\n")
        merges = [tuple(m.split()) for m in merges[1:49152 - 256 - 2 + 1] if len(m.split()) == 2]
        self.byte_encoder = _bytes_to_unicode()
        vocab = list(self.byte_encoder.values())
        vocab = vocab + [v + "</w>" for v in vocab]
        vocab += ["".join(m) for m in merges]
        vocab += ["<|startoftext|>", "<|endoftext|>"]
        self.encoder = {v: i for i, v in enumerate(vocab)}
        self.bpe_ranks = {m: i for i, m in enumerate(merges)}
        self.cache = {"<|startoftext|>": "<|startoftext|>", "<|endoftext|>": "<|endoftext|>"}
        import regex  # \p{L} / \p{N} classes: the pattern of OpenAI clip / open_clip's SimpleTokenizer

        self.pat = regex.compile(
            r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""",
            regex.IGNORECASE)

    def _bpe(self, token):
        if token in self.cache:
            return self.cache[token]
        word = tuple(token[:-1]) + (token[-1] + "</w>",)
        while len(word) > 1:
            pairs = set(zip(word[:-1], word[1:]))
            bigram = min(pairs, key=lambda p: self.bpe_ranks.get(p, float("inf")))
            if bigram not in self.bpe_ranks:
                break
            first, second = bigram
            new, i = [], 0
            while i < len(word):
                if i < len(word) - 1 and word[i] == first and word[i + 1] == second:
                    new.append(first + second)
                    i += 2
                else:
                    new.append(word[i])
                    i += 1
            word = tuple(new)
        out = " ".join(word)
        self.cache[token] = out
        return out

    def encode(self, text):
        text = _whitespace_clean(_basic_clean(text)).lower()
        ids = []
        for tok in self.pat.findall(text):
            tok = "".join(self.byte_encoder[b] for b in tok.encode("utf-8"))
            ids.extend(self.encoder[t] for t in self._bpe(tok).split(" "))
        return ids

    def __call__(self, texts):
        torch = _torch()
        if isinstance(texts, str):
            texts = [texts]
        sot, eot = self.encoder["<|startoftext|>"], self.encoder["<|endoftext|>"]
        out = torch.zeros(len(texts), self.context_length, dtype=torch.long)
        for i, t in enumerate(texts):
            ids = [sot] + self.encode(t) + [eot]
            if len(ids) > self.context_length:
                ids = ids[: self.context_length]
                ids[-1] = eot
            out[i, : len(ids)] = torch.tensor(ids)
        return out


def _basic_clean(text):
    """clip.simple_tokenizer.basic_clean: ftfy.fix_text, then html.unescape twice.  Without ftfy (not
    installable offline) the Unicode NFC normalisation ftfy applies by default is kept; its mojibake repair
    is not reproduced."""
    try:
        import ftfy

        text = ftfy.fix_text(text)
    except ImportError:
        import unicodedata

        text = unicodedata.normalize("NFC", text)
    return html.unescape(html.unescape(text)).strip()


def _whitespace_clean(text):
    import re

    return re.sub(r"\s+", " ", text).strip()


def _bytes_to_unicode():
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(2 ** 8):
        if b not in bs:
            bs.append(b)
            cs.append(2 ** 8 + n)
            n += 1
    return dict(zip(bs, [chr(c) for c in cs]))


def siglip_clean(text):
    """open_clip's `canonicalize_text(basic_clean(text))`, the cleaning of its SigLIP tokenizers: `_` becomes a space,
    ASCII punctuation is removed, the text is lower-cased and its whitespace collapsed."""
    import string

    text = _basic_clean(text).replace("_", " ")
    text = text.translate(str.maketrans("", "", string.punctuation)).lower()
    return " ".join(text.split()).strip()


def siglip_tokenizer(arch, clip_cache_path):
    """open_clip's HFTokenizer of a SigLIP model: `<clip_cache_path>/<arch.tokenizer>/tokenizer.json`, texts cleaned
    by `siglip_clean`, truncated and padded (pad id 1) to the arch's context length; the `_MissingTokenizer` when the
    file is not there."""
    from .xlmr_clip import XLMRTokenizer

    path = os.path.join(clip_cache_path, arch.tokenizer, "tokenizer.json") if clip_cache_path else None
    if path and os.path.exists(path):
        return XLMRTokenizer(path, pad_id=1, context_length=arch.context_length, clean=siglip_clean)
    return _MissingTokenizer("SigLIP tokenizer (%s/tokenizer.json) not found under clip_cache_path" % arch.tokenizer)


class _MissingTokenizer:
    def __init__(self, why):
        self.why = why

    def __call__(self, texts):
        raise RuntimeError(self.why)


# The weight files of a HuggingFace snapshot folder, in the order they are looked for: one file, or the index of a
# sharded snapshot (its "weight_map" names the shard of every tensor), as `save_pretrained` writes large models.
HF_SNAPSHOT_FILES = ("pytorch_model.bin", "model.safetensors", "pytorch_model.bin.index.json",
                     "model.safetensors.index.json")


def _find_checkpoint(key, clip_cache_path):
    """`<clip_cache_path>/<name>.{pt,pth,bin}` with `/`, `@`, `:` of the model name turned into `-`
    (e.g. `ViT-L-14.pt`, `ViT-bigG-14.pt`, `hf_clip-patrickjohncyh-fashion-clip.bin`), or for `hf_clip:` names the
    first of HF_SNAPSHOT_FILES in a HuggingFace snapshot folder `<clip_cache_path>/<repo>/`."""
    if not clip_cache_path:
        return None
    stems = [key.replace("open_clip:", "").replace("/", "-").replace("@", "-").replace(":", "-")]
    if key.startswith("hf_clip:"):
        repo = key[len("hf_clip:"):]
        stems.append(repo.replace("/", "-"))
        for f in HF_SNAPSHOT_FILES:
            p = os.path.join(clip_cache_path, repo, f)
            if os.path.exists(p):
                return p
    for stem in stems:
        for ext in (".pt", ".pth", ".bin"):
            p = os.path.join(clip_cache_path, stem + ext)
            if os.path.exists(p):
                return p
    return None


def _read_tensor_file(path):
    """One weight file: a `.safetensors` file, or anything torch.load / torch.jit.load reads."""
    torch = _torch()
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file

        return load_file(path, device="cpu")
    try:
        return torch.load(path, map_location="cpu", weights_only=False)
    except RuntimeError:
        return torch.jit.load(path, map_location="cpu")


def _read_sharded(index_path):
    """The state_dict of a sharded HuggingFace snapshot: every shard the index's weight_map names, each read once."""
    import json

    with open(index_path) as f:
        weight_map = json.load(f)["weight_map"]
    folder = os.path.dirname(index_path)
    sd = {}
    for shard in sorted(set(weight_map.values())):
        part = _read_tensor_file(os.path.join(folder, shard))
        sd.update((k, part[k]) for k, s in weight_map.items() if s == shard)
    return sd


def read_checkpoint(path, arch):
    """Load a checkpoint file into the OpenAI/open_clip state_dict key layout `load_state_dict` takes.
    Accepted: a plain state_dict, a training checkpoint `{"state_dict": ...}` (optionally with `module.`
    prefixes), a TorchScript archive (OpenAI's released `.pt` files), a HuggingFace CLIPModel state_dict, as one
    `.bin` / `.safetensors` file or as the `*.index.json` of a sharded snapshot."""
    obj = _read_sharded(path) if path.endswith(".index.json") else _read_tensor_file(path)
    sd = obj if isinstance(obj, dict) else obj.state_dict()
    if "state_dict" in sd and isinstance(sd["state_dict"], dict):
        sd = sd["state_dict"]
    if sd and all(k.startswith("module.") for k in sd):
        sd = {k[len("module."):]: v for k, v in sd.items()}
    if any(k.startswith("vision_model.") for k in sd):
        sd = convert_hf_state_dict(sd, arch)
    return sd


@lru_cache(maxsize=None)
def load_clip(clip_model="ViT-B/32", use_jit=True, warmup_batch_size=1, clip_cache_path=None, device=None,
              max_batch=None):
    """Drop-in for all_clip.load_clip (call sites mapper.py:36-41, worker.py:52-57, clip_back.py:868).

    Returns (model, preprocess, tokenizer).  Weights come from `<clip_cache_path>/<model>.pt` (a
    state_dict in the OpenAI/open_clip key layout, or a HuggingFace CLIPModel state_dict); the name
    prefix `synthetic:` selects seeded random weights of that architecture (benchmarks; no network).
    `open_clip:xlm-roberta-base-ViT-B-32` / `open_clip:xlm-roberta-large-ViT-H-14` give a `B200XLMRClip`
    (xlmr_clip.py) and the XLM-R tokenizer of `<clip_cache_path>/xlm-roberta-{base,large}/tokenizer.json`.
    `use_jit` is accepted and ignored (there is no TorchScript path).  Cached per argument tuple like
    the upstream loader, so reader and mapper builders share one model."""
    del use_jit
    from .xlmr_clip import load_xlmr_clip, resolve_xlmr_clip

    torch = _torch()
    xlmr = resolve_xlmr_clip(clip_model)
    arch, key = xlmr if xlmr is not None else resolve_arch(clip_model)
    if device is None:
        dev_index = torch.cuda.current_device() if torch.cuda.is_available() else 0
    else:
        d = torch.device(device)
        if d.type != "cuda":
            raise RuntimeError("b200clip has no CPU path: device=%r" % (device,))
        dev_index = d.index if d.index is not None else torch.cuda.current_device()
    mb = max_batch or max(int(warmup_batch_size), 1)
    if xlmr is not None:
        # open_clip's XLM-RoBERTa CLIPs: an image-only CLIP handle and the text encoder with the MLP head
        return load_xlmr_clip(clip_model, arch, key, warmup_batch_size, clip_cache_path, dev_index, mb)
    model = B200Clip(arch, device=dev_index, max_batch=mb)
    if clip_model.startswith("synthetic:"):
        model.load_state_dict(synthetic_state_dict(arch, seed=0))
    else:
        if key.startswith("nm:"):
            raise NotImplementedError("%r names a DeepSparse quantised ONNX export; this engine loads dense "
                                      "state_dicts (use the open_clip checkpoint of the same architecture)" % clip_model)
        ckpt = _find_checkpoint(key, clip_cache_path)
        if ckpt is None:
            raise FileNotFoundError(
                "no checkpoint for %r under clip_cache_path=%r (no network here); use 'synthetic:%s' for "
                "seeded random weights" % (clip_model, clip_cache_path, clip_model))
        model.load_state_dict(read_checkpoint(ckpt, arch))
    mode, mean, std = preprocess_params(clip_model)
    preprocess = make_preprocess(arch.image_size, mode, mean, std)
    bpe = os.path.join(clip_cache_path, "bpe_simple_vocab_16e6.txt.gz") if clip_cache_path else None
    if isinstance(arch, SigLIPArch):
        tokenizer = siglip_tokenizer(arch, clip_cache_path)
    elif bpe and os.path.exists(bpe):
        tokenizer = SimpleTokenizer(bpe, arch.context_length)
    else:
        tokenizer = _MissingTokenizer("CLIP BPE vocabulary (bpe_simple_vocab_16e6.txt.gz) not found under clip_cache_path")
    # warm-up as upstream does (two forwards on zero inputs): allocates nothing new, primes the kernels
    if warmup_batch_size and torch.cuda.is_available():
        wb = min(int(warmup_batch_size), mb)
        model.embed_image_device(torch.zeros(wb, 3, arch.image_size, arch.image_size, device=model.device))
        toks = torch.zeros(wb, arch.context_length, dtype=torch.long, device=model.device)
        toks[:, 0], toks[:, 1] = arch.vocab_size - 2, arch.vocab_size - 1
        model.embed_text_device(toks)
        torch.cuda.synchronize(model.device)
    return model, preprocess, tokenizer
