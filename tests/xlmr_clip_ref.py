"""CPU restatement of the text tower of open_clip's XLM-RoBERTa CLIPs (`xlm-roberta-base-ViT-B-32`,
`xlm-roberta-large-ViT-H-14`), in plain fp32 torch, on top of tests/mclip_ref.py's encoder.

open_clip's `HFTextEncoder` with `pooler_type: "mean_pooler"` and `proj: "mlp"` (DESIGN §5 (xv)):
  mask = ids != pad_id;  h = XLMRobertaModel(ids, attention_mask=mask).last_hidden_state
  pooled = (h * mask[..., None]).sum(1) / mask.sum(-1, keepdim=True)
  out = Linear(h_mid, D, bias=False)(GELU()(Linear(d, h_mid, bias=False)(pooled))),  h_mid = (d + D) // 2
then clip_back's normalized().  State dicts use mclip_ref's key layout with projection.0.weight [h_mid, d] and
projection.2.weight [D, h_mid] in place of projection.weight: the layout of the GPU text encoder with the MLP head.
PIN: tests/golden/xlmr_clip_tiny.npz holds the same computation by `transformers` XLMRobertaModel (5.5) and a
torch.nn head (tests/golden/make_xlmr_clip_golden.py); tests/test_xlmr_clip_cpu.py checks this file against it.
"""
from dataclasses import replace

import numpy as np
import torch

import mclip_ref

_XLMR = dict(family="xlm-roberta", vocab_size=250002, max_positions=514, type_vocab_size=1, pad_token_id=1, eps=1e-5,
             proj_bias=False)
# name -> (encoder config with out_dim = D, MLP hidden width)
CONFIGS = {
    "xlm-roberta-base-ViT-B-32": (mclip_ref.EncCfg(layers=12, width=768, heads=12, ffn=3072, out_dim=512, **_XLMR), 640),
    "xlm-roberta-large-ViT-H-14": (mclip_ref.EncCfg(layers=24, width=1024, heads=16, ffn=4096, out_dim=1024, **_XLMR),
                                   1024),
    # the golden's shape: head dim 64, 80 positions (77 tokens from position 2), a hidden width with a column tail
    "tiny": (mclip_ref.EncCfg("xlm-roberta", 2, 128, 2, 256, 300, 80, 1, 1, 1e-5, 96, False), 112),
}


def make_state_dict(cfg, hidden, seed=0):
    """mclip_ref's seeded encoder weights and a seeded MLP head (normal, std fan_in ** -0.5)."""
    sd = mclip_ref.make_state_dict(replace(cfg, proj_bias=False), seed)
    del sd["projection.weight"]
    g = torch.Generator().manual_seed(1000 + seed)
    sd["projection.0.weight"] = torch.randn(hidden, cfg.width, generator=g) * cfg.width ** -0.5
    sd["projection.2.weight"] = torch.randn(cfg.out_dim, hidden, generator=g) * hidden ** -0.5
    return sd


def lengths_of(ids, pad_id):
    """Token counts of right-padded rows: mask.sum(-1)."""
    return (np.asarray(ids) != pad_id).sum(1).astype(np.int32)


@torch.no_grad()
def head(sd, pooled):
    """The MLP head on pooled rows fp32 [B, d]."""
    y = torch.nn.functional.gelu(pooled @ sd["projection.0.weight"].t())
    return y @ sd["projection.2.weight"].t()


@torch.no_grad()
def features(sd, cfg, ids):
    """Raw fp32 features [B, D] of right-padded ids [B, T] (open_clip's encode_text before the norm)."""
    lengths = lengths_of(ids, cfg.pad_token_id)
    h = mclip_ref.hidden(sd, cfg, ids, lengths)
    m = torch.as_tensor(np.asarray(ids) != cfg.pad_token_id).float()
    pooled = (h * m[:, :, None]).sum(1) / m.sum(-1, keepdim=True)
    return head(sd, pooled).numpy()


def embeddings(sd, cfg, ids):
    """What the mapper / query service keep: normalized() fp32 rows [B, D]."""
    return mclip_ref.normalized(features(sd, cfg, ids)).astype(np.float32)
