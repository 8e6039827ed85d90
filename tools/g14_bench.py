#!/usr/bin/env python
"""ViT-g-14 and ViT-bigG-14 against ViT-H/14 on seeded random weights of the real sizes, in one run.

  python tools/g14_bench.py [--batches 256,1024] [--text-batch 1024] [--iters 3] [--json OUT]

- image towers of g-14, bigG and H/14 through `embed_image_device` (device fp32 [B, 3, 224, 224] in, normalised fp16
  out) at each of --batches: images/s, and useful TFLOP/s from the shapes, 2 T L (4 w^2 + 2 w mlp) per image (the
  layer GEMMs; attention, 2-3 % of the flops, and the patch embedding are left out);
- the text towers through `embed_text_device` at --text-batch full-length captions: captions/s;
- the attention share of the image forward's device time at the largest batch, from the handle's span timer (a
  separate profiled call);
- ms per batch-1 `encode_image` on device input, replayed from the handle's CUDA graph (median of 50 calls).
One model is resident at a time.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NAMES = ("open_clip:ViT-H-14", "open_clip:ViT-g-14", "open_clip:ViT-bigG-14")


def tower_gflop(t, T):
    """Layer-GEMM GFLOP per sample of a tower: 2 T L (4 w^2 + 2 w mlp)."""
    return 2.0 * T * t.layers * (4 * t.width ** 2 + 2 * t.width * t.mlp) / 1e9


def _timed(fn, iters):
    import torch

    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def bench_one(name, batches, text_batch, iters):
    import numpy as np
    import torch
    import clip_retrieval_b200 as m

    arch, _ = m.model.resolve_arch(name)
    mb = max(max(batches), text_batch)
    model = m.B200Clip(arch, device=0, max_batch=mb).load_state_dict(m.synthetic_state_dict(arch, seed=0))
    S = arch.image_size
    T = (S // arch.patch) ** 2 + 1
    gf_img = tower_gflop(arch.vision, T)
    r = {"name": name, "vision": vars(arch.vision), "text": vars(arch.text), "image_tokens": T,
         "image_gflop_per_sample": gf_img, "image": {}}
    gen = torch.Generator(device="cuda").manual_seed(0)
    px = torch.randn(max(batches), 3, S, S, device="cuda", generator=gen)
    for B in batches:
        x = px[:B]
        s = _timed(lambda: model.embed_image_device(x), iters)
        r["image"][B] = {"ms": s * 1e3, "images_per_s": B / s, "tflops": B * gf_img / s / 1e3}

    model.set_profiling(True)
    model.embed_image_device(px)
    torch.cuda.synchronize()
    tm = model.last_timing()
    model.set_profiling(False)
    total = tm["gemm"] + tm["attention"] + tm["layernorm"] + tm["other"]
    r["timing_batch"] = max(batches)
    r["timing"] = tm
    r["attention_share"] = tm["attention"] / total if total else None

    tok = torch.randint(1, arch.vocab_size - 2, (text_batch, arch.context_length), device="cuda", generator=gen)
    tok[:, 0], tok[:, -1] = arch.vocab_size - 2, arch.vocab_size - 1
    s = _timed(lambda: model.embed_text_device(tok), iters)
    gf_txt = tower_gflop(arch.text, arch.context_length)
    r["text"] = dict(r["text"], batch=text_batch, ms=s * 1e3, captions_per_s=text_batch / s,
                     tflops=text_batch * gf_txt / s / 1e3)

    x1 = px[:1].contiguous()
    for _ in range(3):                                      # eager, capture, first replay
        model.encode_image(x1)
    lat = []
    for _ in range(50):
        torch.cuda.synchronize()
        t = time.perf_counter()
        model.encode_image(x1)
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t) * 1e3)
    r["b1_ms_median"], r["b1_ms_min"] = float(np.median(lat)), float(np.min(lat))
    del model
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="256,1024")
    ap.add_argument("--text-batch", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("g14_bench.py needs a CUDA device")
    batches = [int(b) for b in args.batches.split(",")]
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power, "models": []}
    print("%s, power limit %s" % (out["device"], power))
    for name in NAMES:
        r = bench_one(name, batches, args.text_batch, args.iters)
        out["models"].append(r)
        v, t, tm = r["vision"], r["text"], r["timing"]
        print("%s: image %d x %d / %d heads (hd %d), %.0f GFLOP per image" % (
            name, v["width"], v["layers"], v["heads"], v["width"] // v["heads"], r["image_gflop_per_sample"]))
        for B, x in r["image"].items():
            print("  image batch %5d: %8.1f images/s  %6.1f ms  %6.1f TFLOP/s" % (B, x["images_per_s"], x["ms"],
                                                                                x["tflops"]))
        print("  image batch %d device time: gemm %.1f (qkv %.1f, out_proj %.1f, fc %.1f, c_proj %.1f), attention %.1f "
              "(%.1f %%), layernorm %.1f, other %.1f ms" % (
                  r["timing_batch"], tm["gemm"], tm["gemm_by_kind"]["qkv"], tm["gemm_by_kind"]["out_proj"],
                  tm["gemm_by_kind"]["fc"], tm["gemm_by_kind"]["c_proj"], tm["attention"],
                  100 * (r["attention_share"] or 0), tm["layernorm"], tm["other"]))
        print("  text batch %d: %.1f captions/s (%.1f ms, %.1f TFLOP/s)" % (t["batch"], t["captions_per_s"], t["ms"],
                                                                           t["tflops"]))
        print("  encode_image batch 1 (graph): median %.3f ms, min %.3f ms" % (r["b1_ms_median"], r["b1_ms_min"]))
    h = out["models"][0]["image"]
    for r in out["models"][1:]:
        print("%s / ViT-H-14 useful image TFLOP/s: %s" % (r["name"], ", ".join(
            "batch %d %.2f" % (B, r["image"][B]["tflops"] / h[B]["tflops"]) for B in batches)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
