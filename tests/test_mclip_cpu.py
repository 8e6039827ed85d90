"""Host side of the multilingual text towers (use_mclip): the fp32 oracle against the HuggingFace goldens, the
tokenizer wrapper against the ids `PreTrainedTokenizerFast` returns under the reference's call arguments, the
M-CLIP / SentenceTransformer folder readers, and the error cases."""
import json
import os

import numpy as np
import pytest
import torch

import mclip_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def write_mclip_folder(path, sd, cfg, safetensors=False):
    """An M-CLIP folder (MultilingualCLIP.save_pretrained layout) holding the oracle weights `sd`."""
    os.makedirs(path, exist_ok=True)
    raw = {("LinearTransformation." + k[len("projection."):] if k.startswith("projection.") else "transformer." + k): v
           for k, v in sd.items()}
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({"model_type": "M-CLIP", "modelBase": "xlm-roberta-large", "transformerDimensions": cfg.width,
                   "numDims": cfg.out_dim}, f)
    _save(raw, path, safetensors)


def write_st_folder(path, sd, cfg, max_seq_length=128, pooling="mean", activation="Identity", safetensors=False):
    """A SentenceTransformer folder: DistilBERT module at the root, 1_Pooling, 2_Dense."""
    from clip_retrieval_b200.mclip import _DISTILBERT_NAMES

    os.makedirs(os.path.join(path, "1_Pooling"), exist_ok=True)
    os.makedirs(os.path.join(path, "2_Dense"), exist_ok=True)
    model = {}
    for k, v in sd.items():
        if k.startswith("projection."):
            continue
        if k.startswith("encoder.layer."):
            i, rest = k[len("encoder.layer."):].split(".", 1)
            for a, b in _DISTILBERT_NAMES:
                if rest.startswith(b + "."):
                    rest = a + rest[len(b):]
                    break
            k = "transformer.layer.%s.%s" % (i, rest)
        model[k] = v
    _save(model, path, safetensors)
    dense = {"linear.weight": sd["projection.weight"]}
    if "projection.bias" in sd:
        dense["linear.bias"] = sd["projection.bias"]
    _save(dense, os.path.join(path, "2_Dense"), False)
    files = {
        "modules.json": [{"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
                         {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
                         {"idx": 2, "name": "2", "path": "2_Dense", "type": "sentence_transformers.models.Dense"}],
        "sentence_bert_config.json": {"max_seq_length": max_seq_length, "do_lower_case": False},
        "config.json": {"model_type": "distilbert", "n_layers": cfg.layers, "dim": cfg.width, "n_heads": cfg.heads,
                        "hidden_dim": cfg.ffn, "vocab_size": cfg.vocab_size,
                        "max_position_embeddings": cfg.max_positions, "pad_token_id": cfg.pad_token_id,
                        "sinusoidal_pos_embds": False, "activation": "gelu"},
        "1_Pooling/config.json": {"word_embedding_dimension": cfg.width, "pooling_mode_cls_token": pooling == "cls",
                                  "pooling_mode_mean_tokens": pooling == "mean", "pooling_mode_max_tokens": False},
        "2_Dense/config.json": {"in_features": cfg.width, "out_features": cfg.out_dim,
                                "bias": "projection.bias" in sd,
                                "activation_function": "torch.nn.modules.%s" % (
                                    "linear.Identity" if activation == "Identity" else "activation." + activation)},
    }
    for name, obj in files.items():
        with open(os.path.join(path, name), "w") as f:
            json.dump(obj, f)


def _save(sd, folder, safetensors):
    sd = {k: v.contiguous() for k, v in sd.items()}
    if safetensors:
        from safetensors.torch import save_file

        save_file(sd, os.path.join(folder, "model.safetensors"))
    else:
        torch.save(sd, os.path.join(folder, "pytorch_model.bin"))


@pytest.mark.parametrize("name", ["tiny-xlmr", "tiny-distilbert"])
def test_oracle_matches_hf_golden(name):
    cfg = mclip_ref.CONFIGS[name]
    z = np.load(os.path.join(GOLDEN, "mclip_%s.npz" % name))
    assert len(set(z["lengths"].tolist())) > 3 and z["lengths"].min() == 1     # ragged, including a single token
    got = mclip_ref.features(mclip_ref.make_state_dict(cfg, seed=0), cfg, z["ids"], z["lengths"])
    np.testing.assert_allclose(got, z["features"], rtol=1e-5, atol=1e-5)


def test_oracle_ignores_padding():
    cfg = mclip_ref.CONFIGS["tiny-xlmr"]
    sd = mclip_ref.make_state_dict(cfg, seed=0)
    ids = mclip_ref.synth_ids([5, 9], cfg)
    padded = np.concatenate([ids, np.full((2, 7), cfg.pad_token_id)], 1)
    np.testing.assert_allclose(mclip_ref.features(sd, cfg, padded, [5, 9]), mclip_ref.features(sd, cfg, ids, [5, 9]),
                               rtol=1e-5, atol=1e-6)
    zero = mclip_ref.normalized(np.zeros((2, 4), np.float32))
    assert np.array_equal(zero, np.zeros((2, 4)))


def _golden_tokens():
    with open(os.path.join(GOLDEN, "mclip_tokenizer_golden.json")) as f:
        return json.load(f)


def _check_tokens(got, want):
    ids, lengths = got
    want_ids, mask = np.array(want["input_ids"]), np.array(want["attention_mask"])
    assert np.array_equal(ids, want_ids) and ids.dtype == np.int64
    assert np.array_equal(lengths, mask.sum(1)) and lengths.dtype == np.int32
    assert np.array_equal(np.arange(ids.shape[1])[None, :] < lengths[:, None], mask.astype(bool))   # right padding


def test_tokenizer_unigram_matches_pretrained_tokenizer_fast():
    pytest.importorskip("tokenizers")
    from clip_retrieval_b200.mclip import MCLIP_ARCHS, MclipTokenizer

    g = _golden_tokens()
    tok = MclipTokenizer(os.path.join(GOLDEN, "mclip_unigram_tokenizer.json"),
                         MCLIP_ARCHS["M-CLIP/XLM-Roberta-Large-Vit-L-14"])
    _check_tokens(tok(g["texts"]), g["unigram"]["batch"])        # pad id 1, no truncation
    _check_tokens(tok([g["texts"][1]]), g["unigram"]["single"])
    assert (tok(g["texts"])[0] == 1).any()
    with pytest.raises(ValueError, match="positions"):
        tok(["the " * 600])                                      # > 512 tokens: M-CLIP itself would fail


def test_tokenizer_wordpiece_truncates_like_sentence_transformers():
    pytest.importorskip("tokenizers")
    from dataclasses import replace
    from clip_retrieval_b200.mclip import MCLIP_ARCHS, MclipTokenizer

    g = _golden_tokens()
    arch = replace(MCLIP_ARCHS["sentence-transformers/clip-ViT-B-32-multilingual-v1"],
                   max_seq_length=g["st_max_seq_length"])
    ids, lengths = MclipTokenizer(os.path.join(GOLDEN, "mclip_wordpiece_tokenizer.json"), arch)(g["texts"])
    _check_tokens((ids, lengths), g["wordpiece"])                # pad id 0, truncation at max_seq_length
    assert lengths.max() == g["st_max_seq_length"] and ids[lengths.argmax(), lengths.max() - 1] == 3   # [SEP] kept


@pytest.mark.parametrize("safetensors", [False, True])
@pytest.mark.parametrize("bias", [False, True])
def test_st_folder_reader(tmp_path, bias, safetensors):
    from clip_retrieval_b200.mclip import resolve_mclip

    cfg = mclip_ref.CONFIGS["tiny-distilbert"]
    sd = mclip_ref.make_state_dict(cfg, seed=1)
    if bias:
        sd["projection.bias"] = torch.randn(cfg.out_dim)
    write_st_folder(str(tmp_path), sd, cfg, max_seq_length=24, safetensors=safetensors)
    arch, got, folder = resolve_mclip(str(tmp_path))
    assert folder == str(tmp_path)
    assert (arch.family, arch.layers, arch.width, arch.heads, arch.ffn, arch.out_dim) == (
        "distilbert", cfg.layers, cfg.width, cfg.heads, cfg.ffn, cfg.out_dim)
    assert arch.layer_norm_eps == 1e-12 and arch.position_offset == 0 and arch.type_vocab_size == 0
    assert arch.max_seq_length == 24 and arch.proj_bias == bias
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)


@pytest.mark.parametrize("safetensors", [False, True])
def test_mclip_folder_reader_and_cache_names(tmp_path, safetensors):
    from clip_retrieval_b200.mclip import resolve_mclip

    cfg = mclip_ref.CONFIGS["tiny-xlmr"]
    sd = mclip_ref.make_state_dict(cfg, seed=2)
    repo = "M-CLIP/XLM-Roberta-Large-Vit-B-32"
    for sub in (repo, repo.replace("/", "-")):
        cache = tmp_path / sub.replace("/", "_")
        write_mclip_folder(str(cache / sub), sd, cfg, safetensors=safetensors)
        arch, got, folder = resolve_mclip(repo, str(cache))
        assert folder == str(cache / sub)
        assert (arch.family, arch.layers, arch.width, arch.heads, arch.ffn, arch.vocab_size, arch.max_positions) == (
            "xlm-roberta", cfg.layers, cfg.width, cfg.heads, cfg.ffn, cfg.vocab_size, cfg.max_positions)
        assert arch.layer_norm_eps == 1e-5 and arch.position_offset == 2 and arch.type_vocab_size == 1
        assert arch.out_dim == cfg.out_dim and arch.proj_bias and arch.max_seq_length == 0
        assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)


def test_error_cases(tmp_path):
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.mclip import load_mclip, resolve_mclip

    for name in ("x", "synthetic:x", "M-CLIP/unknown"):
        with pytest.raises(NotImplementedError, match="accepted"):
            resolve_mclip(name)
    with pytest.raises(NotImplementedError):
        m.ClipMapper(True, True, False, True, "synthetic:ViT-B/32", True, "x")
    with pytest.raises(FileNotFoundError):
        resolve_mclip("M-CLIP/XLM-Roberta-Large-Vit-L-14", str(tmp_path))
    with pytest.raises(ValueError, match="not available"):
        load_mclip("ViT-Z/99")
    cfg = mclip_ref.CONFIGS["tiny-distilbert"]
    sd = mclip_ref.make_state_dict(cfg, seed=1)
    write_st_folder(str(tmp_path / "cls"), sd, cfg, pooling="cls")
    with pytest.raises(NotImplementedError, match="mean pooling"):
        resolve_mclip(str(tmp_path / "cls"))
    write_st_folder(str(tmp_path / "tanh"), sd, cfg, activation="Tanh")
    with pytest.raises(NotImplementedError, match="Identity"):
        resolve_mclip(str(tmp_path / "tanh"))
    svc = m.B200KnnService({"x": m.ClipResource(model=None, device="cuda")})
    with pytest.raises(ValueError, match="model_txt_mclip"):
        svc.query(text_input="ein Hund", use_mclip=True)


def test_real_size_arch_table():
    from clip_retrieval_b200.mclip import CLIP_TO_MCLIP, MCLIP_ARCHS

    x = MCLIP_ARCHS[CLIP_TO_MCLIP["ViT-L/14"]]
    assert (x.layers, x.width, x.heads, x.ffn, x.vocab_size, x.max_positions, x.out_dim) == (
        24, 1024, 16, 4096, 250002, 514, 768)
    assert x.layer_norm_eps == 1e-5 and x.max_tokens == 512 and x.proj_bias
    assert MCLIP_ARCHS[CLIP_TO_MCLIP["ViT-B/32"]].out_dim == 512
    d = MCLIP_ARCHS["sentence-transformers/clip-ViT-B-32-multilingual-v1"]
    assert (d.layers, d.width, d.heads, d.ffn, d.out_dim, d.max_seq_length, d.proj_bias) == (6, 768, 12, 3072, 512,
                                                                                                  128, False)
    for k, c in (("xlmr-large", x), ("distilbert-multilingual", d)):
        r = mclip_ref.CONFIGS[k]
        assert (r.layers, r.width, r.heads, r.ffn, r.vocab_size, r.max_positions, r.eps) == (
            c.layers, c.width, c.heads, c.ffn, c.vocab_size, c.max_positions, c.layer_norm_eps)
