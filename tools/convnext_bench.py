#!/usr/bin/env python
"""The six ConvNeXt CLIP image towers (arch, px) on seeded random weights of the real sizes, and ViT-H/14 for
comparison, in one run.

  python tools/convnext_bench.py [--batch 256] [--iters 3] [--models convnext_base,...] [--json OUT]

Per model:
- images/s through `embed_image_device` (device fp32 [B, 3, S, S] in, normalised fp16 out) at --batch;
- useful TFLOP/s from the trunk's MACs per image (trunk_gmacs below: the stem, the depthwise 7x7 taps, fc1 / fc2, the
  downsamples; the head and LayerNorms are not counted), 2 FLOP per MAC;
- the device-time split between dwconv7_ln, the 1x1 GEMMs (fc1, fc2, the stem), ln_s2d + the downsample GEMMs and the
  head, from a separate torch.profiler run of one batch (the downsample GEMM runs the same kernel as fc1 / fc2 and is
  counted with the GEMMs);
- dwconv7_ln alone at the stage-0 and stage-1 shapes of the batch, in GB/s over its required bytes (the input read
  once, the output written once, the fp32 weights once), against the 3.35 TB/s data-sheet figure;
- ms per batch-1 `encode_image`, replayed from the handle's CUDA graph (median of 50 calls);
- the same forward through torch.nn.functional in bf16 with channels_last (cuDNN depthwise convolution + cuBLAS), on
  the same weights, as a reference rate measured in the same call.
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

NAMES = ("convnext_base", "convnext_base_w", "convnext_base_w_320", "convnext_large_d", "convnext_large_d_320",
         "convnext_xxlarge")
HBM_TBS = 3.35   # H100 SXM data sheet


def trunk_gmacs(a):
    """Multiply-accumulates per image of the trunk, in G."""
    g = a.image_size // 4
    f = g * g * 48 * a.dims[0]
    for s, (n, C) in enumerate(zip(a.depths, a.dims)):
        H = g >> s
        if s > 0:
            f += H * H * 4 * a.dims[s - 1] * C
        f += n * H * H * (49 * C + 8 * C * C)
    return f / 1e9


def torch_forward(sd, a, px):
    """The image tower in bf16 through torch.nn.functional (cuDNN depthwise convolution, cuBLAS linears,
    channels_last)."""
    import torch
    import torch.nn.functional as F

    t, eps = "visual.trunk.", a.eps

    def ln_c(x, p):
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), sd[p + ".weight"], sd[p + ".bias"], eps).permute(0, 3, 1, 2)

    x = px.bfloat16().contiguous(memory_format=torch.channels_last)
    x = ln_c(F.conv2d(x, sd[t + "stem.0.weight"], sd[t + "stem.0.bias"], stride=4), t + "stem.1")
    for s, n in enumerate(a.depths):
        p = "%sstages.%d." % (t, s)
        if s > 0:
            x = F.conv2d(ln_c(x, p + "downsample.0"), sd[p + "downsample.1.weight"], sd[p + "downsample.1.bias"], stride=2)
        for j in range(n):
            b = "%sblocks.%d." % (p, j)
            C = x.shape[1]
            y = F.conv2d(x, sd[b + "conv_dw.weight"], sd[b + "conv_dw.bias"], padding=3, groups=C).permute(0, 2, 3, 1)
            y = F.layer_norm(y, (C,), sd[b + "norm.weight"], sd[b + "norm.bias"], eps)
            y = F.linear(F.gelu(F.linear(y, sd[b + "mlp.fc1.weight"], sd[b + "mlp.fc1.bias"])), sd[b + "mlp.fc2.weight"],
                         sd[b + "mlp.fc2.bias"])
            x = x + (y * sd[b + "gamma"]).permute(0, 3, 1, 2)
    pooled = F.layer_norm(x.float().mean((2, 3)), (x.shape[1],), sd[t + "head.norm.weight"].float(),
                          sd[t + "head.norm.bias"].float(), eps)
    if a.head_mlp:
        f = F.linear(F.gelu(F.linear(pooled, sd["visual.head.mlp.fc1.weight"].float(),
                                     sd["visual.head.mlp.fc1.bias"].float())), sd["visual.head.mlp.fc2.weight"].float())
    else:
        f = F.linear(pooled, sd["visual.head.proj.weight"].float())
    return (f / f.norm(dim=-1, keepdim=True)).half()


def _timed(fn, iters):
    import torch

    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def _split(model, px):
    """Device ms per kernel class over one profiled forward."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.embed_image_device(px)
        torch.cuda.synchronize()
    cls = {"dwconv7_ln": 0.0, "gemm": 0.0, "ln_s2d": 0.0, "head": 0.0, "other": 0.0}
    for e in prof.key_averages():
        name = e.key
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        t /= 1e3
        if "dwconv7_ln" in name:
            cls["dwconv7_ln"] += t
        elif "gemm_bf16_wgmma" in name:
            cls["gemm"] += t
        elif "ln_s2d" in name:
            cls["ln_s2d"] += t
        elif "mean_ln_rows" in name or "mlp" in name or "feat_norm" in name:
            cls["head"] += t
        elif "Memcpy" not in name and "Memset" not in name:
            cls["other"] += t
    return cls


def _dwconv_gbs(B, H, C):
    """dwconv7_ln alone on [B, H, H, C]: GB/s over its required bytes, median of 10 timed calls (CUDA events)."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    x = torch.randn(B, H, H, C, device="cuda").bfloat16()
    out = torch.empty_like(x)
    w = torch.randn(49, C, device="cuda") / 7
    b, g, be = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def run():
        check(lib.b200_dwconv7_ln_bf16_device(x.data_ptr(), B, H, H, C, w.data_ptr(), b.data_ptr(), g.data_ptr(),
                                              be.data_ptr(), 1e-6, out.data_ptr(), 0, st), "dwconv7_ln")

    run()
    ts = []
    for _ in range(10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    ts.sort()
    nbytes = 2 * 2 * B * H * H * C + 4 * 52 * C
    return nbytes / ts[len(ts) // 2] / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--models", default=",".join(NAMES))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import clip_retrieval_b200 as m

    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power, "batch": args.batch, "models": []}
    print("%s, power limit %s" % (out["device"], power))
    B = args.batch
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name in args.models.split(","):
        a = m.CONVNEXT_ARCHS["open_clip:" + name]
        sd = m.synthetic_state_dict(a, seed=0)
        model = m.B200Clip(a, device=0, max_batch=B).load_state_dict(sd)
        px = torch.randn(B, 3, a.image_size, a.image_size, device="cuda", generator=gen).clamp_(-1.8, 2.15)
        dt = _timed(lambda: model.embed_image_device(px), args.iters)
        split = _split(model, px)
        one = px[:1].contiguous()
        for _ in range(3):
            model.encode_image(one)
        lat = []
        for _ in range(50):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.encode_image(one)
            torch.cuda.synchronize()
            lat.append((time.perf_counter() - t0) * 1e3)
        ours = model.embed_image_device(px)
        del model
        torch.cuda.empty_cache()
        g0 = a.image_size // 4
        gbs = [_dwconv_gbs(B, g0 >> s, a.dims[s]) for s in (0, 1)]
        torch.cuda.empty_cache()
        sdc = {k: v.bfloat16().cuda() for k, v in sd.items() if k.startswith("visual.")}
        with torch.no_grad():
            dt_ref = _timed(lambda: torch_forward(sdc, a, px), args.iters)
            ref = torch_forward(sdc, a, px)
        cos = float((ours.float() * ref.float()).sum(-1).min())
        del sdc
        torch.cuda.empty_cache()
        gm = trunk_gmacs(a)
        r = {"model": name, "px": a.image_size, "images_per_s": B / dt, "trunk_gmacs_per_image": gm,
             "tflops": 2 * gm * B / dt / 1e3, "split_ms": split, "dwconv7_ln_gbs_stage0_1": gbs,
             "batch1_ms_median": float(np.median(lat)), "torch_bf16_images_per_s": B / dt_ref,
             "min_cos_vs_torch": cos}
        out["models"].append(r)
        tot = sum(split.values()) or 1.0
        print("%-20s %3d px %7.0f img/s  %6.1f TFLOP/s (%.2f GMAC/img)  dwconv7_ln %4.1f%%  GEMM %4.1f%%  ln_s2d %4.1f%%  "
              "head %4.1f%%  other %4.1f%%  dwconv7_ln s0/s1 %.0f / %.0f GB/s (%.0f%% / %.0f%% of %.2f TB/s)  batch-1 "
              "%.2f ms  torch bf16 %7.0f img/s  (min cos vs torch %.4f)"
              % (name, a.image_size, r["images_per_s"], r["tflops"], gm, 100 * split["dwconv7_ln"] / tot,
                 100 * split["gemm"] / tot, 100 * split["ln_s2d"] / tot, 100 * split["head"] / tot,
                 100 * split["other"] / tot, gbs[0], gbs[1], gbs[0] / HBM_TBS / 10, gbs[1] / HBM_TBS / 10, HBM_TBS,
                 r["batch1_ms_median"], r["torch_bf16_images_per_s"], cos))
        sys.stdout.flush()
    # ViT-H/14 in the same run, for comparison
    a = m.ARCHS["open_clip:ViT-H-14"]
    model = m.B200Clip(a, device=0, max_batch=B).load_state_dict(m.synthetic_state_dict(a, seed=0))
    px = torch.randn(B, 3, 224, 224, device="cuda", generator=gen)
    dt = _timed(lambda: model.embed_image_device(px), args.iters)
    one = px[:1].contiguous()
    for _ in range(3):
        model.encode_image(one)
    lat = []
    for _ in range(50):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.encode_image(one)
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t0) * 1e3)
    out["vit_h14"] = {"images_per_s": B / dt, "batch1_ms_median": float(np.median(lat))}
    print("%-20s %3d px %7.0f img/s  batch-1 %.2f ms" % ("ViT-H-14", 224, B / dt, float(np.median(lat))))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
