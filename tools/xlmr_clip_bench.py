"""open_clip's XLM-RoBERTa CLIPs on one GPU, synthetic weights of the real sizes.

  * mapper: `embed_text` (the mapper's host-buffer call: ids [1024, 77] in, fp16 rows out) at batch 1024 with caption
    lengths drawn uniformly from 8..40 tokens, for xlm-roberta-base-ViT-B-32 and xlm-roberta-large-ViT-H-14:
    captions per second;
  * query service: the large text tower at batch 1 (`embed_text_device` on a [1, 77] CUDA row, lengths 8, 16, 32):
    wall time per query (host clock around a device synchronise).
Work per token from the shapes: the layer GEMMs are 2 (4 w^2 + 2 w ffn) flop per token per layer, i.e. 170 MFLOP
(base) and 604 MFLOP (large) per token, plus 4 len w flop of attention per token per layer.
One JSON line per measurement; the card name, power limit and max SM clock go with them.

    python tools/xlmr_clip_bench.py [--iters 100] [--out results/xlmr_clip_bench.jsonl]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mclip_bench import card, timed  # noqa: E402


def caption_ids(B, lo, hi, seed):
    """Right-padded ids [B, 77]: <s>, random ids, </s>, then pad 1, with lengths uniform in lo..hi."""
    import numpy as np

    rng = np.random.default_rng(seed)
    ids = np.full((B, 77), 1, dtype=np.int64)
    lens = rng.integers(lo, hi + 1, size=B)
    for i, n in enumerate(lens):
        ids[i, :n] = rng.integers(5, 250002, size=n)
        ids[i, 0], ids[i, n - 1] = 0, 2
    return ids, lens


def layer_gemm_flop_per_token(t):
    return 2 * t.layers * (4 * t.width * t.width + 2 * t.width * t.ffn)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.xlmr_clip import XLMR_CLIP_ARCHS, synthetic_state_dict

    assert torch.cuda.is_available(), "xlmr_clip_bench needs a GPU"
    lines = []
    dev = card()

    def emit(rec):
        rec["card"] = dev
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    B = 1024
    for name in ("xlm-roberta-base-ViT-B-32", "xlm-roberta-large-ViT-H-14"):
        arch = XLMR_CLIP_ARCHS[name]
        model = m.B200XLMRClip(arch, device=0, max_batch=B).load_state_dict(synthetic_state_dict(arch, seed=0))
        ids, lens = caption_ids(B, 8, 40, 1)
        s = timed(lambda: model.embed_text(ids), max(10, a.iters // 10))
        emit({"what": name + " mapper embed_text", "batch": B, "tokens_per_caption": "8..40 (mean %.1f)" % lens.mean(),
              "captions_per_s": round(B / s, 1), "ms_per_batch": round(s * 1e3, 3),
              "layer_gemm_mflop_per_token": round(layer_gemm_flop_per_token(arch.text) / 1e6, 1)})
        if name.startswith("xlm-roberta-large"):
            for L in (8, 16, 32):
                one, _ = caption_ids(1, L, L, L)
                d_one = torch.as_tensor(one).cuda()
                ms = timed(lambda: model.embed_text_device(d_one, dtype=torch.float32), a.iters) * 1e3
                emit({"what": name + " query", "batch": 1, "T": 77, "tokens": L, "ms_per_query": round(ms, 4)})
        del model
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
