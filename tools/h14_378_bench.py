#!/usr/bin/env python
"""ViT-H/14 at 378 px (`open_clip:ViT-H-14-378-quickgelu`, seeded random weights): the image tower as `ClipMapper`
calls it and as a batch-1 query runs.

  python tools/h14_378_bench.py [--batch 256] [--iters 5] [--json OUT]

- images/s of `embed_image` (host fp32 [B, 3, 378, 378] in, normalised fp16 out: H2D, forward, D2H) at --batch;
- ms per batch-1 `encode_image` on device input, replayed from the handle's CUDA graph (median of 50 calls);
- the attention share of the batch forward's device time, from the handle's span timer (a separate profiled call).
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NAME = "synthetic:open_clip:ViT-H-14-378-quickgelu"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    import clip_retrieval_b200 as m

    if not torch.cuda.is_available():
        raise SystemExit("h14_378_bench.py needs a CUDA device")
    arch, _ = m.model.resolve_arch(NAME)
    model = m.B200Clip(arch, device=0, max_batch=args.batch).load_state_dict(m.synthetic_state_dict(arch, seed=0))
    S, B = arch.image_size, args.batch
    px = torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(0)).numpy()

    model.embed_image(px)                                   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.iters):
        model.embed_image(px)                               # returns after the D2H copy
    batch_s = (time.perf_counter() - t0) / args.iters

    model.set_profiling(True)
    model.embed_image(px)
    tm = model.last_timing()
    model.set_profiling(False)
    total = tm["gemm"] + tm["attention"] + tm["layernorm"] + tm["other"]

    x1 = torch.from_numpy(px[:1]).cuda()
    for _ in range(3):                                      # eager, capture, first replay
        model.encode_image(x1)
    lat = []
    for _ in range(50):
        torch.cuda.synchronize()
        t = time.perf_counter()
        model.encode_image(x1)
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t) * 1e3)

    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    r = {"device": torch.cuda.get_device_name(0), "power_limit": power, "batch": B,
         "images_per_s": B / batch_s, "batch_ms": batch_s * 1e3, "b1_ms_median": float(np.median(lat)),
         "b1_ms_min": float(np.min(lat)), "attention_ms": tm["attention"], "device_ms": total,
         "attention_share": tm["attention"] / total if total else None, "timing": tm}
    print("%s, power limit %s" % (r["device"], power))
    print("embed_image batch %d: %.1f images/s (%.1f ms per batch); attention %.1f of %.1f ms device time (%.1f %%)"
          % (B, r["images_per_s"], r["batch_ms"], tm["attention"], total, 100 * (r["attention_share"] or 0)))
    print("encode_image batch 1 (graph): median %.3f ms, min %.3f ms" % (r["b1_ms_median"], r["b1_ms_min"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
