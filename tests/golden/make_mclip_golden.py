"""Regenerate the multilingual text-tower goldens (needs `transformers` and `tokenizers`; run from the repository
root: `python tests/golden/make_mclip_golden.py`).

mclip_<config>.npz: ids, lengths and the raw features (masked mean pool + projection) that HuggingFace
XLMRobertaModel / DistilBertModel compute on the seeded weights of tests/mclip_ref.py, for the tiny configs, with
ragged lengths.
mclip_wordpiece_tokenizer.json / mclip_unigram_tokenizer.json: a tiny WordPiece (BERT-style, [CLS] .. [SEP], pad 0)
and a tiny Unigram + Metaspace (XLM-R-style, <s> .. </s>, pad 1) tokenizer.  mclip_tokenizer_golden.json: the ids
and attention masks `PreTrainedTokenizerFast` returns for them under the reference's call arguments:
  M-CLIP: tokenizer(texts, padding=True, return_tensors="pt")
  SentenceTransformer: tokenizer(texts, padding=True, truncation="longest_first", return_tensors="pt",
                                 max_length=max_seq_length)
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import mclip_ref  # noqa: E402

LENGTHS = [1, 7, 19, 2, 33, 12]
TEXTS = ["a cat on the mat", "un chat sur le tapis", "ein Hund", "", "the the the the the the the the the the the "
         "the the the the the the the the the the the the the the the the the the the the the the the the the", "x"]
ST_MAX_SEQ = 16


def to_hf(sd, cfg):
    if cfg.family == "xlm-roberta":
        return {k: v for k, v in sd.items() if not k.startswith("projection.")}
    out = {}
    for k, v in sd.items():
        if k.startswith("projection."):
            continue
        if k.startswith("encoder.layer."):
            i, rest = k[len("encoder.layer."):].split(".", 1)
            rest = (rest.replace("attention.self.query", "attention.q_lin").replace("attention.self.key", "attention.k_lin")
                    .replace("attention.self.value", "attention.v_lin").replace("attention.output.dense", "attention.out_lin")
                    .replace("attention.output.LayerNorm", "sa_layer_norm").replace("intermediate.dense", "ffn.lin1")
                    .replace("output.dense", "ffn.lin2").replace("output.LayerNorm", "output_layer_norm"))
            k = "transformer.layer.%s.%s" % (i, rest)
        out[k] = v
    return out


def hf_features(name):
    from transformers import DistilBertConfig, DistilBertModel, XLMRobertaConfig, XLMRobertaModel

    cfg = mclip_ref.CONFIGS[name]
    sd = mclip_ref.make_state_dict(cfg, seed=0)
    if cfg.family == "xlm-roberta":
        hc = XLMRobertaConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.width, num_hidden_layers=cfg.layers,
                              num_attention_heads=cfg.heads, intermediate_size=cfg.ffn,
                              max_position_embeddings=cfg.max_positions, type_vocab_size=cfg.type_vocab_size,
                              pad_token_id=cfg.pad_token_id, layer_norm_eps=cfg.eps, hidden_dropout_prob=0.0,
                              attention_probs_dropout_prob=0.0, attn_implementation="eager")
        model = XLMRobertaModel(hc, add_pooling_layer=False)
    else:
        hc = DistilBertConfig(vocab_size=cfg.vocab_size, dim=cfg.width, n_layers=cfg.layers, n_heads=cfg.heads,
                              hidden_dim=cfg.ffn, max_position_embeddings=cfg.max_positions,
                              pad_token_id=cfg.pad_token_id, dropout=0.0, attention_dropout=0.0,
                              attn_implementation="eager")
        model = DistilBertModel(hc)
    missing, unexpected = model.load_state_dict(to_hf(sd, cfg), strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    model.eval()
    ids = mclip_ref.synth_ids(LENGTHS, cfg, seed=1)
    lengths = np.array(LENGTHS, dtype=np.int32)
    mask = torch.as_tensor(np.arange(ids.shape[1])[None, :] < lengths[:, None]).long()
    with torch.no_grad():
        h = model(input_ids=torch.as_tensor(ids), attention_mask=mask).last_hidden_state
        pooled = (h * mask[:, :, None]).sum(1) / mask.sum(1, keepdim=True)
        f = pooled @ sd["projection.weight"].t()
        if "projection.bias" in sd:
            f = f + sd["projection.bias"]
    np.savez_compressed(os.path.join(HERE, "mclip_%s.npz" % name), ids=ids, lengths=lengths,
                        features=f.numpy().astype(np.float32))


def tokenizers_golden():
    from tokenizers import Tokenizer, models, normalizers, pre_tokenizers, decoders, processors
    from transformers import PreTrainedTokenizerFast

    words = sorted(set(" ".join(TEXTS).lower().split()))
    # WordPiece: [PAD] 0, [UNK] 1, [CLS] 2, [SEP] 3, then whole words and a few pieces
    vocab = {"[PAD]": 0, "[UNK]": 1, "[CLS]": 2, "[SEP]": 3}
    for t in words + ["##s", "##e", "ch", "##at", "h", "##und"]:
        vocab.setdefault(t, len(vocab))
    wp = Tokenizer(models.WordPiece(vocab, unk_token="[UNK]"))
    wp.normalizer = normalizers.BertNormalizer(lowercase=True)
    wp.pre_tokenizer = pre_tokenizers.BertPreTokenizer()
    wp.post_processor = processors.TemplateProcessing(single="[CLS] $A [SEP]", special_tokens=[("[CLS]", 2), ("[SEP]", 3)])
    wp.decoder = decoders.WordPiece()
    wp.save(os.path.join(HERE, "mclip_wordpiece_tokenizer.json"))
    # Unigram + Metaspace: <s> 0, <pad> 1, </s> 2, <unk> 3
    pieces = [("<s>", 0.0), ("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0)]
    for t in words:
        pieces.append(("▁" + t, -2.0 - 0.1 * len(t)))
    for ch in sorted(set("".join(words))):
        pieces.append((ch, -8.0))
        pieces.append(("▁" + ch, -9.0))
    ug = Tokenizer(models.Unigram(pieces, unk_id=3, byte_fallback=False))
    ug.normalizer = normalizers.NFKC()
    ug.pre_tokenizer = pre_tokenizers.Metaspace()
    ug.post_processor = processors.TemplateProcessing(single="<s> $A </s>", special_tokens=[("<s>", 0), ("</s>", 2)])
    ug.decoder = decoders.Metaspace()
    ug.save(os.path.join(HERE, "mclip_unigram_tokenizer.json"))

    out = {"texts": TEXTS, "st_max_seq_length": ST_MAX_SEQ}
    tw = PreTrainedTokenizerFast(tokenizer_file=os.path.join(HERE, "mclip_wordpiece_tokenizer.json"),
                                 pad_token="[PAD]", unk_token="[UNK]")
    r = tw(TEXTS, padding=True, truncation="longest_first", return_tensors="pt", max_length=ST_MAX_SEQ)
    out["wordpiece"] = {"input_ids": r["input_ids"].tolist(), "attention_mask": r["attention_mask"].tolist()}
    tu = PreTrainedTokenizerFast(tokenizer_file=os.path.join(HERE, "mclip_unigram_tokenizer.json"),
                                 pad_token="<pad>", unk_token="<unk>")
    out["unigram"] = {}
    for key, texts in (("batch", TEXTS), ("single", [TEXTS[1]])):
        r = tu(texts, padding=True, return_tensors="pt")
        out["unigram"][key] = {"input_ids": r["input_ids"].tolist(), "attention_mask": r["attention_mask"].tolist()}
    with open(os.path.join(HERE, "mclip_tokenizer_golden.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    for name in ("tiny-xlmr", "tiny-distilbert"):
        hf_features(name)
    tokenizers_golden()
    print("written under", HERE)
