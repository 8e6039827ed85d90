"""Host side of open_clip's XLM-RoBERTa CLIPs: the fp32 oracle against the HuggingFace golden, the tokenizer against
`PreTrainedTokenizerFast` under open_clip's call, the checkpoint split, the architecture table, name resolution and
the refusals."""
import os
from dataclasses import replace

import numpy as np
import pytest
import torch

import xlmr_clip_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden():
    return np.load(os.path.join(GOLDEN, "xlmr_clip_tiny.npz"))


def tiny_arch():
    """An XLMRClipArch small enough for CPU tests: a one-layer 32 px ViT and the oracle's tiny text tower."""
    import clip_retrieval_b200 as m

    cfg, hidden = xlmr_clip_ref.CONFIGS["tiny"]
    vision = m.ClipArch(cfg.out_dim, 32, 16, m.Tower(64, 1, 1, 128), m.Tower(0, 0, 0, 0), quick_gelu=False)
    text = m.EncoderArch(cfg.family, cfg.layers, cfg.width, cfg.heads, cfg.ffn, cfg.vocab_size, cfg.max_positions,
                         cfg.type_vocab_size, cfg.pad_token_id, cfg.eps, cfg.out_dim, False)
    return m.XLMRClipArch(vision, text, hidden, "xlm-roberta-base")


def open_clip_state_dict(arch, text_sd, seed=0):
    """An open_clip-layout state dict: seeded visual.* tensors, `text_sd` (oracle layout) under text.transformer.* /
    text.proj.*, the keys the loader ignores, and logit_scale."""
    from clip_retrieval_b200.model import synthetic_state_dict

    full = synthetic_state_dict(replace(arch.vision, text=arch.vision.vision), seed)
    sd = {k: v for k, v in full.items() if k.startswith("visual.")}
    for k, v in text_sd.items():
        sd["text.proj" + k[len("projection"):] if k.startswith("projection.") else "text.transformer." + k] = v
    sd["text.transformer.pooler.dense.weight"] = torch.zeros(arch.text.width, arch.text.width)
    sd["text.transformer.pooler.dense.bias"] = torch.zeros(arch.text.width)
    sd["text.transformer.embeddings.position_ids"] = torch.arange(arch.text.max_positions)[None]
    sd["logit_scale"] = torch.tensor(4.6052)
    return sd


def test_oracle_matches_hf_golden():
    z = _golden()
    cfg, hidden = xlmr_clip_ref.CONFIGS["tiny"]
    lengths = xlmr_clip_ref.lengths_of(z["ids"], cfg.pad_token_id)
    assert len(set(lengths.tolist())) > 4 and lengths.max() == 77 and lengths.min() == 2   # ragged, one truncated
    got = xlmr_clip_ref.features(xlmr_clip_ref.make_state_dict(cfg, hidden, seed=0), cfg, z["ids"])
    np.testing.assert_allclose(got, z["features"], rtol=1e-5, atol=1e-5)


def test_tokenizer_matches_pretrained_tokenizer_fast():
    pytest.importorskip("tokenizers")
    from clip_retrieval_b200.xlmr_clip import XLMRTokenizer

    z = _golden()
    tok = XLMRTokenizer(os.path.join(GOLDEN, "mclip_unigram_tokenizer.json"))
    ids = tok([str(t) for t in z["texts"]])
    assert ids.dtype == torch.int64 and tuple(ids.shape) == (len(z["texts"]), 77)
    assert np.array_equal(ids.numpy(), z["ids"])
    long_row = ids[int(np.argmax((z["ids"] != 1).sum(1)))]
    assert int(long_row[-1]) == 2 and int(long_row[0]) == 0           # truncated at 77 with </s> last
    assert np.array_equal(tok(str(z["texts"][0])).numpy(), z["ids"][:1])
    # whitespace cleaning: the spaced-out caption tokenizes as the plain one
    assert torch.equal(tok(["  a   cat\n\ton  the   mat  "]), tok(["a cat on the mat"]))


def test_right_padded_lengths_and_refusals():
    from clip_retrieval_b200.xlmr_clip import right_padded_lengths

    z = _golden()
    assert np.array_equal(right_padded_lengths(z["ids"], 1), xlmr_clip_ref.lengths_of(z["ids"], 1))
    bad = z["ids"].copy()
    bad[2, 40] = 7
    with pytest.raises(ValueError, match="row 2"):
        right_padded_lengths(bad, 1)
    bad = z["ids"].copy()
    bad[5, :] = 1
    with pytest.raises(ValueError, match="row 5 is all padding"):
        right_padded_lengths(bad, 1)


def test_checkpoint_splits_bit_for_bit(tmp_path):
    from clip_retrieval_b200.xlmr_clip import read_xlmr_checkpoint, split_state_dict

    arch = tiny_arch()
    cfg, hidden = xlmr_clip_ref.CONFIGS["tiny"]
    text_sd = xlmr_clip_ref.make_state_dict(cfg, hidden, seed=3)
    sd = open_clip_state_dict(arch, text_sd)
    torch.save(sd, str(tmp_path / "xlm-roberta-base-ViT-B-32.pt"))
    for src in (sd, read_xlmr_checkpoint("open_clip:xlm-roberta-base-ViT-B-32", str(tmp_path), arch)):
        visual, text = split_state_dict(src, arch)
        assert set(visual) == {k for k in sd if k.startswith("visual.")}
        assert all(torch.equal(visual[k], sd[k]) for k in visual)
        assert set(text) == set(text_sd) and all(torch.equal(text[k], text_sd[k]) for k in text)


def test_checkpoint_refusals_name_the_key(tmp_path):
    from clip_retrieval_b200.xlmr_clip import read_xlmr_checkpoint, split_state_dict

    arch = tiny_arch()
    cfg, hidden = xlmr_clip_ref.CONFIGS["tiny"]
    sd = open_clip_state_dict(arch, xlmr_clip_ref.make_state_dict(cfg, hidden, seed=3))
    for key in ("visual.proj", "text.proj.2.weight", "text.transformer.encoder.layer.1.output.dense.bias"):
        broken = dict(sd)
        del broken[key]
        with pytest.raises(ValueError, match="%r is missing" % key):
            split_state_dict(broken, arch)
        broken[key] = torch.zeros(3, 5)
        with pytest.raises(ValueError, match="%r has shape" % key):
            split_state_dict(broken, arch)
    with pytest.raises(FileNotFoundError, match="xlm-roberta"):
        read_xlmr_checkpoint("open_clip:xlm-roberta-base-ViT-B-32", str(tmp_path), arch)


def test_real_size_arch_table():
    from clip_retrieval_b200.model import ARCHS
    from clip_retrieval_b200.xlmr_clip import XLMR_CLIP_ARCHS

    b, h = XLMR_CLIP_ARCHS["xlm-roberta-base-ViT-B-32"], XLMR_CLIP_ARCHS["xlm-roberta-large-ViT-H-14"]
    for x, clip, D, hid, tokdir in ((b, "open_clip:ViT-B-32", 512, 640, "xlm-roberta-base"),
                                    (h, "open_clip:ViT-H-14", 1024, 1024, "xlm-roberta-large")):
        assert x.vision == replace(ARCHS[clip], text=x.vision.text) and not x.vision.quick_gelu
        assert tuple(x.vision.text.__dict__.values()) == (0, 0, 0, 0)
        assert (x.embed_dim, x.image_size, x.hidden, x.tokenizer, x.context_length) == (D, 224, hid, tokdir, 77)
        assert x.hidden == (x.text.width + D) // 2
        t = x.text
        assert (t.family, t.vocab_size, t.max_positions, t.type_vocab_size, t.pad_token_id, t.layer_norm_eps,
                t.out_dim, t.proj_bias, t.position_offset) == ("xlm-roberta", 250002, 514, 1, 1, 1e-5, D, False, 2)
    assert (b.vision.vision.width, b.vision.vision.layers, b.vision.vision.heads, b.vision.vision.mlp,
            b.vision.patch) == (768, 12, 12, 3072, 32)
    assert (h.vision.vision.width, h.vision.vision.layers, h.vision.vision.width // h.vision.vision.heads,
            h.vision.vision.mlp, h.vision.patch) == (1280, 32, 80, 5120, 14)
    assert (b.text.layers, b.text.width, b.text.heads, b.text.ffn) == (12, 768, 12, 3072)
    assert (h.text.layers, h.text.width, h.text.heads, h.text.ffn) == (24, 1024, 16, 4096)
    for name, x in XLMR_CLIP_ARCHS.items():
        r, hid = xlmr_clip_ref.CONFIGS[name]
        assert (r.layers, r.width, r.heads, r.ffn, r.vocab_size, r.max_positions, r.eps, r.out_dim, hid) == (
            x.text.layers, x.text.width, x.text.heads, x.text.ffn, x.text.vocab_size, x.text.max_positions,
            x.text.layer_norm_eps, x.text.out_dim, x.hidden)


def test_name_resolution():
    from clip_retrieval_b200.model import ARCHS, resolve_arch
    from clip_retrieval_b200.xlmr_clip import XLMR_CLIP_ARCHS, resolve_xlmr_clip

    for name in ("open_clip:xlm-roberta-base-ViT-B-32", "open_clip:xlm-roberta-base-ViT-B-32/laion5b_s13b_b90k",
                 "synthetic:open_clip:xlm-roberta-base-ViT-B-32"):
        assert resolve_xlmr_clip(name) == (XLMR_CLIP_ARCHS["xlm-roberta-base-ViT-B-32"],
                                           "open_clip:xlm-roberta-base-ViT-B-32")
    for name in ("open_clip:xlm-roberta-large-ViT-H-14/frozen_laion5b_s13b_b90k",
                 "synthetic:open_clip:xlm-roberta-large-ViT-H-14"):
        assert resolve_xlmr_clip(name)[0] is XLMR_CLIP_ARCHS["xlm-roberta-large-ViT-H-14"]
    # every other name is left to resolve_arch, which resolves as before and refuses unknown ones
    for name in list(ARCHS) + ["open_clip:ViT-B-32/openai", "synthetic:ViT-L/14", "hf_clip:openai/clip-vit-base-patch32"]:
        assert resolve_xlmr_clip(name) is None
        resolve_arch(name)
    for name in ("open_clip:xlm-roberta-huge-ViT-Z-99", "open_clip:xlm-roberta-base-ViT-B-16/laion"):
        assert resolve_xlmr_clip(name) is None
        with pytest.raises(ValueError, match="unknown clip_model"):
            resolve_arch(name)


def test_load_clip_refusals(tmp_path):
    import clip_retrieval_b200 as m

    with pytest.raises(ValueError, match="unknown clip_model"):
        m.load_clip("open_clip:xlm-roberta-base-ViT-B-16", clip_cache_path=str(tmp_path))
    with pytest.raises(FileNotFoundError, match="synthetic:"):         # before any device memory is taken
        m.load_clip("open_clip:xlm-roberta-large-ViT-H-14/frozen_laion5b_s13b_b90k", clip_cache_path=str(tmp_path))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            m.load_clip("synthetic:open_clip:xlm-roberta-base-ViT-B-32", device="cpu")
