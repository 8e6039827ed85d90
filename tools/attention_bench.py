#!/usr/bin/env python
"""Per-shape timing of the attention entry point b200_attention_bf16_device (CUDA events around one CUDA graph of
many launches).

  python tools/attention_bench.py [--iters N] [--json OUT]

For each shape it prints ms per launch, useful TFLOP/s (4 T^2 hd per head, halved for causal), padded TFLOP/s (the
MMA work of the head-dim-64 wgmma kernel: 64-row query tiles, 64-key blocks, the last block of a tile narrowed to
16-column steps; head dim 64 at T <= 320 only) and HBM GB/s (qkv read once, output written once).  Shapes: both
ViT-L/14 towers at batch 1024, the ViT-B/16 and ViT-B/32 image towers, the ViT-H/14 text tower at its serving batches,
and head dim 80: the ViT-H/14-378 image tower (T 730, streaming kernel) at batch 1, 8 and 256 against T 576, the
longest sequence the whole-K/V kernel takes, at batch 256.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, B, T, heads, causal, head dim)
SHAPES = [
    ("ViT-L/14 image", 1024, 257, 16, 0, 64),
    ("ViT-L/14 text", 1024, 77, 12, 1, 64),
    ("ViT-B/16 image", 1024, 197, 12, 0, 64),
    ("ViT-B/32 image", 1024, 50, 12, 0, 64),
    ("ViT-H/14 text b1", 1, 77, 16, 1, 64),
    ("ViT-H/14 text b8", 8, 77, 16, 1, 64),
    ("ViT-H/14 text b64", 64, 77, 16, 1, 64),
    ("H/14-378 image b1", 1, 730, 16, 0, 80),
    ("H/14-378 image b8", 8, 730, 16, 0, 80),
    ("H/14-378 image b256", 256, 730, 16, 0, 80),
    ("hd80 T576 b256", 256, 576, 16, 0, 80),
]


def useful_flops(B, T, heads, causal, hd):
    f = 4.0 * T * T * hd * heads * B
    return f / 2 if causal else f


def padded_flops(B, T, heads, causal, hd):
    if hd != 64 or T > 320:   # the wgmma kernel's work; other shapes run on mma.sync
        return None
    HD = hd
    cols = 0
    for t in range((T + 63) // 64):
        kend = min(T, 64 * t + 64) if causal else T
        nkt = (kend + 63) // 64
        cols += 64 * (nkt - 1) + 16 * ((kend - 64 * (nkt - 1) + 15) // 16)
    return 2 * 2 * 64 * cols * HD * heads * B   # S and P V, 64 query rows per tile


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    import clip_retrieval_b200  # noqa: F401
    from clip_retrieval_b200._lib import lib, check

    if not torch.cuda.is_available():
        raise SystemExit("attention_bench.py needs a CUDA device")
    rows = []
    st = torch.cuda.current_stream().cuda_stream
    for name, B, T, heads, causal, hd in SHAPES:
        w = heads * hd
        g = torch.Generator(device="cuda").manual_seed(T + B)
        qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
        out = torch.empty(B * T, w, device="cuda", dtype=torch.bfloat16)

        def run(s=st):
            check(lib.b200_attention_bf16_device(qkv.data_ptr(), out.data_ptr(), B, T, heads, w, causal, 0, s), "attention")

        for _ in range(5):
            run()
        iters = args.iters if B >= 64 else args.iters * 20
        # the launches are captured into one CUDA graph: at the serving batches a kernel takes a few microseconds, less
        # than the host needs to issue it, so timing eager launches would time the host
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cap = torch.cuda.current_stream().cuda_stream
            for _ in range(iters):
                run(cap)
        graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        byts = B * T * 4 * w * 2
        pf = padded_flops(B, T, heads, causal, hd)
        r = {"shape": name, "B": B, "T": T, "heads": heads, "causal": causal, "hd": hd, "ms": ms,
             "useful_tflops": useful_flops(B, T, heads, causal, hd) / (ms / 1e3) / 1e12,
             "padded_tflops": None if pf is None else pf / (ms / 1e3) / 1e12,
             "hbm_gbs": byts / (ms / 1e3) / 1e9}
        rows.append(r)
        padded = "   n/a" if pf is None else "%6.1f" % r["padded_tflops"]
        print("%-19s B=%-5d T=%-4d heads=%-3d hd=%-3d causal=%d  %9.4f ms  useful %6.1f TFLOP/s  padded %s TFLOP/s  "
              "%7.1f GB/s" % (name, B, T, heads, hd, causal, ms, r["useful_tflops"], padded, r["hbm_gbs"]))
        del qkv, out
    props = torch.cuda.get_device_properties(0)
    power = _power_limit()
    print("device: %s, power limit %s" % (props.name, power))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": props.name, "power_limit": power, "rows": rows}, f, indent=1)


def _power_limit():
    import subprocess

    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


if __name__ == "__main__":
    main()
