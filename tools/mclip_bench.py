"""Multilingual text towers (use_mclip) on one GPU, synthetic weights of the real sizes.

  * query service: M-CLIP XLM-RoBERTa-Large (24 layers, width 1024) at batch 1, T = 8, 16, 32, 64 tokens: wall time
    per query (host clock around a device synchronise), then the device time per kernel class and the launch count
    from a separate profiled run;
  * mapper: the multilingual DistilBERT (6 layers, width 768) at batch 256, T = 32: captions per second.
One JSON line per measurement; the card name and power limit go with them.

    python tools/mclip_bench.py [--iters 200] [--out results/mclip_bench.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return "unknown (%s)" % e


def ids_for(arch, B, T, seed):
    import numpy as np

    rng = np.random.default_rng(seed)
    ids = rng.integers(5, arch.vocab_size, size=(B, T)).astype(np.int64)
    return ids, np.full(B, T, dtype=np.int32)


def timed(fn, iters):
    import torch

    for _ in range(max(3, iters // 10)):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.mclip import MCLIP_ARCHS, synthetic_state_dict

    assert torch.cuda.is_available(), "mclip_bench needs a GPU"
    lines = []
    dev = card()

    def emit(rec):
        rec["card"] = dev
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    arch = MCLIP_ARCHS["M-CLIP/XLM-Roberta-Large-Vit-L-14"]
    enc = m.B200TextEncoder(arch, device=0, max_batch=1, max_tokens=64).load_state_dict(synthetic_state_dict(arch))
    for T in (8, 16, 32, 64):
        ids, lens = ids_for(arch, 1, T, T)
        d_ids, d_len = torch.as_tensor(ids).cuda(), torch.as_tensor(lens).cuda()
        ms = timed(lambda: enc.embed_text_device(d_ids, d_len), a.iters) * 1e3
        enc.set_profiling(True)
        for _ in range(10):
            enc.embed_text_device(d_ids, d_len)
        t = enc.last_timing()
        enc.set_profiling(False)
        split = {k: round(t[k] / 10, 4) for k in ("gemm", "attention", "layernorm", "other")}
        emit({"what": "xlmr-large query", "batch": 1, "T": T, "ms_per_query": round(ms, 4),
              "device_ms_by_class": split, "launches": t["launches"]})
    del enc
    torch.cuda.empty_cache()

    arch = MCLIP_ARCHS["sentence-transformers/clip-ViT-B-32-multilingual-v1"]
    B, T = 256, 32
    enc = m.B200TextEncoder(arch, device=0, max_batch=B, max_tokens=128).load_state_dict(synthetic_state_dict(arch))
    ids, lens = ids_for(arch, B, T, 1)
    d_ids, d_len = torch.as_tensor(ids).cuda(), torch.as_tensor(lens).cuda()
    s = timed(lambda: enc.embed_text_device(d_ids, d_len), max(20, a.iters // 4))
    s_host = timed(lambda: enc.embed_text(ids, lens), max(20, a.iters // 4))
    emit({"what": "distilbert-multilingual mapper", "batch": B, "T": T, "captions_per_s": round(B / s, 1),
          "captions_per_s_host_buffers": round(B / s_host, 1)})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
