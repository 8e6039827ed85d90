"""CPU restatement of the multilingual text towers behind `use_mclip`, in plain fp32 torch.

What it restates:
  * M-CLIP `MultilingualCLIP.forward([text], tokenizer)` (clip_back.py:836-859): XLMRobertaModel last hidden state,
    `(h * mask).sum(1) / mask.sum(1)`, `LinearTransformation` (with bias);
  * SentenceTransformer `encode` of the mapper (mapper.py:44-47,62-63): DistilBertModel, mean pooling
    (`sum / clamp(count, 1e-9)`), Dense without activation;
  each followed by clip_back's `normalized()` (a zero norm divides by 1).
Encoder: embeddings (word + token_type[0]) + position, LayerNorm; per layer x = LN1(x + out(attn(x))),
x = LN2(x + W2 gelu_erf(W1 x)); attention bidirectional, keys past a sample's length masked.  LayerNorm eps from
the config.  Position ids: XLM-R padding_idx + 1 + t for the tokens of a sample (padding_idx for the padding),
DistilBERT t.
State dicts use the HuggingFace BERT / XLM-R key layout without a model prefix, plus projection.{weight,bias}: the
layout b200_text_encoder_load_weights takes.
PIN: tests/golden/mclip_*.npz hold the same computation by `transformers` XLMRobertaModel / DistilBertModel (5.5) on
these seeded weights (tests/golden/make_mclip_golden.py); tests/test_mclip_cpu.py checks this file against them.
"""
from dataclasses import dataclass

import numpy as np
import torch


@dataclass(frozen=True)
class EncCfg:
    family: str            # "xlm-roberta" or "distilbert"
    layers: int
    width: int
    heads: int
    ffn: int
    vocab_size: int
    max_positions: int
    type_vocab_size: int   # 0: no token-type table
    pad_token_id: int
    eps: float
    out_dim: int
    proj_bias: bool

    @property
    def position_offset(self):
        return self.pad_token_id + 1 if self.family == "xlm-roberta" else 0


CONFIGS = {
    "xlmr-large": EncCfg("xlm-roberta", 24, 1024, 16, 4096, 250002, 514, 1, 1, 1e-5, 768, True),
    "distilbert-multilingual": EncCfg("distilbert", 6, 768, 12, 3072, 119547, 512, 0, 0, 1e-12, 512, False),
    # small shapes for the goldens and fast tests (same structure, head dim 64)
    "tiny-xlmr": EncCfg("xlm-roberta", 2, 128, 2, 256, 300, 40, 1, 1, 1e-5, 96, True),
    "tiny-distilbert": EncCfg("distilbert", 2, 192, 3, 384, 300, 40, 0, 0, 1e-12, 64, False),
}


def make_state_dict(cfg, seed=0):
    """Seeded weights at BERT's init scale (normal, std 0.02) with non-trivial LayerNorm affine and biases."""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std=0.02):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    w = cfg.width
    sd = {"embeddings.word_embeddings.weight": rn(cfg.vocab_size, w),
          "embeddings.position_embeddings.weight": rn(cfg.max_positions, w)}
    if cfg.type_vocab_size:
        sd["embeddings.token_type_embeddings.weight"] = rn(cfg.type_vocab_size, w)
    sd["embeddings.LayerNorm.weight"] = 1.0 + rn(w, std=0.1)
    sd["embeddings.LayerNorm.bias"] = rn(w, std=0.05)
    for i in range(cfg.layers):
        p = "encoder.layer.%d." % i
        for n in ("query", "key", "value"):
            sd[p + "attention.self.%s.weight" % n] = rn(w, w)
            sd[p + "attention.self.%s.bias" % n] = rn(w)
        sd[p + "attention.output.dense.weight"] = rn(w, w)
        sd[p + "attention.output.dense.bias"] = rn(w)
        sd[p + "attention.output.LayerNorm.weight"] = 1.0 + rn(w, std=0.1)
        sd[p + "attention.output.LayerNorm.bias"] = rn(w, std=0.05)
        sd[p + "intermediate.dense.weight"] = rn(cfg.ffn, w)
        sd[p + "intermediate.dense.bias"] = rn(cfg.ffn)
        sd[p + "output.dense.weight"] = rn(w, cfg.ffn)
        sd[p + "output.dense.bias"] = rn(w)
        sd[p + "output.LayerNorm.weight"] = 1.0 + rn(w, std=0.1)
        sd[p + "output.LayerNorm.bias"] = rn(w, std=0.05)
    sd["projection.weight"] = rn(cfg.out_dim, w, std=w ** -0.5)
    if cfg.proj_bias:
        sd["projection.bias"] = rn(cfg.out_dim)
    return sd


def synth_ids(lengths, cfg, seed=0):
    """Right-padded ids [B, max(lengths)] (int64) as the tokenizers produce them: a start id, random ids, an end id,
    then the pad id.  XLM-R: <s> 0, </s> 2; DistilBERT-style: 101 / 102 (clamped into a small vocabulary)."""
    rng = np.random.default_rng(3000 + seed)
    T = int(max(lengths))
    if cfg.family == "xlm-roberta":
        start, end = 0, 2
    else:
        start, end = min(101, cfg.vocab_size - 2), min(102, cfg.vocab_size - 1)
    ids = np.full((len(lengths), T), cfg.pad_token_id, dtype=np.int64)
    for i, n in enumerate(lengths):
        ids[i, :n] = rng.integers(5, cfg.vocab_size, size=n)
        ids[i, 0] = start
        if n > 1:
            ids[i, n - 1] = end
    return ids


def _ln(x, sd, p, eps):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], eps)


@torch.no_grad()
def hidden(sd, cfg, ids, lengths):
    """Last hidden state fp32 [B, T, w] of right-padded ids [B, T] with per-sample lengths."""
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long)
    B, T = ids.shape
    lengths = torch.as_tensor(np.asarray(lengths), dtype=torch.long)
    mask = torch.arange(T)[None, :] < lengths[:, None]
    if cfg.family == "xlm-roberta":
        pos = torch.where(mask, cfg.pad_token_id + 1 + torch.arange(T)[None, :], torch.tensor(cfg.pad_token_id))
    else:
        pos = torch.arange(T)[None, :].expand(B, T)
    x = sd["embeddings.word_embeddings.weight"][ids]
    if cfg.type_vocab_size:
        x = x + sd["embeddings.token_type_embeddings.weight"][0]
    x = x + sd["embeddings.position_embeddings.weight"][pos]
    x = _ln(x, sd, "embeddings.LayerNorm", cfg.eps)
    w, H = cfg.width, cfg.heads
    hd = w // H
    bias = torch.zeros(B, 1, 1, T).masked_fill(~mask[:, None, None, :], float("-inf"))
    for i in range(cfg.layers):
        p = "encoder.layer.%d." % i

        def lin(t, n):
            return t @ sd[p + n + ".weight"].t() + sd[p + n + ".bias"]

        q, k, v = (lin(x, "attention.self." + n).view(B, T, H, hd).transpose(1, 2) for n in ("query", "key", "value"))
        a = torch.softmax((q @ k.transpose(-1, -2)) * hd ** -0.5 + bias, -1) @ v
        a = a.transpose(1, 2).reshape(B, T, w)
        x = _ln(x + lin(a, "attention.output.dense"), sd, p + "attention.output.LayerNorm", cfg.eps)
        f = torch.nn.functional.gelu(lin(x, "intermediate.dense"))
        x = _ln(x + lin(f, "output.dense"), sd, p + "output.LayerNorm", cfg.eps)
    return x


@torch.no_grad()
def features(sd, cfg, ids, lengths):
    """Masked mean pool + projection: the raw fp32 features [B, D] (M-CLIP's forward / ST's encode)."""
    h = hidden(sd, cfg, ids, lengths)
    T = h.shape[1]
    lengths = torch.as_tensor(np.asarray(lengths), dtype=torch.long)
    m = (torch.arange(T)[None, :] < lengths[:, None]).float()
    pooled = (h * m[:, :, None]).sum(1) / m.sum(1, keepdim=True)
    out = pooled @ sd["projection.weight"].t()
    if "projection.bias" in sd:
        out = out + sd["projection.bias"]
    return out.numpy()


def normalized(a, axis=-1, order=2):
    """clip_back.py:194-197 / mapper.py:8-13."""
    l2 = np.atleast_1d(np.linalg.norm(a, order, axis))
    l2[l2 == 0] = 1
    return a / np.expand_dims(l2, axis)


def embeddings(sd, cfg, ids, lengths):
    """What the mapper / query service keep: normalized() fp32 rows [B, D]."""
    return normalized(features(sd, cfg, ids, lengths)).astype(np.float32)


def cosine(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return (a * b).sum(-1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))
