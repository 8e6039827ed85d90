"""Regenerate tests/golden/xlmr_clip_tiny.npz (needs `transformers` and `tokenizers`; run from the repository root:
`python tests/golden/make_xlmr_clip_golden.py`).

texts: captions, some with extra whitespace and HTML entities, one longer than 77 tokens, one empty.
ids [n, 77]: what open_clip's HFTokenizer returns for them with the tiny Unigram tokenizer of
mclip_unigram_tokenizer.json: each text cleaned by whitespace_clean(basic_clean(.)) (ftfy left out: NFC
normalisation only), then PreTrainedTokenizerFast(texts, max_length=77, padding="max_length", truncation=True).
features [n, D]: HuggingFace XLMRobertaModel on the seeded weights of tests/xlmr_clip_ref.py ("tiny"), open_clip's
mean pool under mask = ids != pad, and a torch.nn Sequential(Linear, GELU, Linear) head without biases.
"""
import html
import os
import re
import sys
import unicodedata

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import xlmr_clip_ref  # noqa: E402

TEXTS = ["a cat on the mat", "un chat sur le tapis", "ein Hund", "", " ".join(["the"] * 100), "x",
         "  a   cat\n\ton  the   mat  ", "le chat &amp;amp; le Hund", "the cat the mat the hund " * 2]


def clean(text):
    text = html.unescape(html.unescape(unicodedata.normalize("NFC", text))).strip()
    return re.sub(r"\s+", " ", text).strip()


def main():
    from transformers import PreTrainedTokenizerFast, XLMRobertaConfig, XLMRobertaModel

    tok = PreTrainedTokenizerFast(tokenizer_file=os.path.join(HERE, "mclip_unigram_tokenizer.json"),
                                  pad_token="<pad>", unk_token="<unk>")
    ids = tok([clean(t) for t in TEXTS], max_length=77, padding="max_length", truncation=True,
              return_tensors="pt")["input_ids"]
    cfg, hidden = xlmr_clip_ref.CONFIGS["tiny"]
    sd = xlmr_clip_ref.make_state_dict(cfg, hidden, seed=0)
    hc = XLMRobertaConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.width, num_hidden_layers=cfg.layers,
                          num_attention_heads=cfg.heads, intermediate_size=cfg.ffn,
                          max_position_embeddings=cfg.max_positions, type_vocab_size=cfg.type_vocab_size,
                          pad_token_id=cfg.pad_token_id, layer_norm_eps=cfg.eps, hidden_dropout_prob=0.0,
                          attention_probs_dropout_prob=0.0, attn_implementation="eager")
    model = XLMRobertaModel(hc, add_pooling_layer=False)
    missing, unexpected = model.load_state_dict({k: v for k, v in sd.items() if not k.startswith("projection.")},
                                                strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    model.eval()
    proj = torch.nn.Sequential(torch.nn.Linear(cfg.width, hidden, bias=False), torch.nn.GELU(),
                               torch.nn.Linear(hidden, cfg.out_dim, bias=False))
    proj[0].weight.data.copy_(sd["projection.0.weight"])
    proj[2].weight.data.copy_(sd["projection.2.weight"])
    with torch.no_grad():
        mask = (ids != cfg.pad_token_id).long()
        h = model(input_ids=ids, attention_mask=mask).last_hidden_state
        pooled = (h * mask.unsqueeze(-1)).sum(1) / mask.sum(-1, keepdim=True)
        f = proj(pooled)
    np.savez_compressed(os.path.join(HERE, "xlmr_clip_tiny.npz"), texts=np.array(TEXTS), ids=ids.numpy(),
                        features=f.numpy().astype(np.float32))
    print("written", os.path.join(HERE, "xlmr_clip_tiny.npz"))


if __name__ == "__main__":
    main()
