#!/usr/bin/env python
"""The five ResNet CLIP image towers on seeded random weights of the real sizes, in one run.

  python tools/resnet_bench.py [--batch 256] [--iters 3] [--models RN50,RN101,...] [--json OUT]

Per model:
- images/s through `embed_image_device` (device fp32 [B, 3, S, S] in, normalised fp16 out) at --batch;
- useful TFLOP/s from the convolution and GEMM shapes (conv_gflop below: every convolution with its true Cin, the
  attention-pool projections of all T tokens, c_proj of token 0; the padding of the implicit convolution's channels
  to 64 is not counted);
- the device-time split between the implicit 3x3 convolutions (conv3x3_bf16_wgmma_kernel), the 1x1 GEMMs (the other
  wgmma GEMM kernels, the attention pool's q / k / v projection included), the pools and gathers, and the attention
  pool's attention and c_proj tail, from a separate torch.profiler run of one batch;
- ms per batch-1 `encode_image` on device input, replayed from the handle's CUDA graph (median of 50 calls);
- the same forward through cuDNN (torch.nn.functional in bf16, channels_last, the same folded weights), as a reference
  rate measured in the same call.
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

NAMES = ("RN50", "RN101", "RN50x4", "RN50x16", "RN50x64")


def conv_gflop(a):
    """Useful GFLOP per image of the image tower's convolutions and GEMMs."""
    w, S = a.width, a.image_size
    g = S // 2
    f = 2.0 * g * g * (27 * (w // 2) + 9 * (w // 2) ** 2 + 9 * (w // 2) * w)
    H, cin = S // 4, w
    for s, n in enumerate(a.layers):
        p = w << s
        for j in range(n):
            stride = 2 if (j == 0 and s > 0) else 1
            Ho = H // stride
            f += 2.0 * (H * H * (cin * p + 9 * p * p) + Ho * Ho * p * 4 * p)
            if stride > 1 or cin != 4 * p:
                f += 2.0 * Ho * Ho * cin * 4 * p
            cin, H = 4 * p, Ho
    C, T = 32 * w, H * H + 1
    f += 2.0 * T * 3 * C * C + 2.0 * C * a.embed_dim
    return f / 1e9


def folded(sd, a):
    """The BatchNorm-folded weights (fp64 fold, bf16 / fp32 storage as the library keeps them), as torch tensors."""
    import torch

    out = {}

    def fold(conv, bn):
        sc = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + 1e-5)
        out[conv] = (sd[conv + ".weight"].double() * sc[:, None, None, None]).bfloat16().cuda()
        out[conv + ".b"] = (sd[bn + ".bias"].double() - sd[bn + ".running_mean"].double() * sc).float().cuda()

    fold("visual.conv1", "visual.bn1")
    fold("visual.conv2", "visual.bn2")
    fold("visual.conv3", "visual.bn3")
    for s, n in enumerate(a.layers):
        for j in range(n):
            p = "visual.layer%d.%d." % (s + 1, j)
            for i in (1, 2, 3):
                fold(p + "conv%d" % i, p + "bn%d" % i)
            if p + "downsample.0.weight" in sd:
                fold(p + "downsample.0", p + "downsample.1")
    at = "visual.attnpool."
    for k in ("positional_embedding", "q_proj.weight", "k_proj.weight", "v_proj.weight", "c_proj.weight"):
        out[at + k] = sd[at + k].bfloat16().cuda()
    for k in ("q_proj.bias", "k_proj.bias", "v_proj.bias", "c_proj.bias"):
        out[at + k] = sd[at + k].float().cuda()
    return out


def cudnn_forward(fw, a, px):
    """The image tower in bf16 through torch.nn.functional (cuDNN convolutions, channels_last)."""
    import torch
    import torch.nn.functional as F

    def cv(x, k, stride=1, pad=0):
        return F.conv2d(x, fw[k], fw[k + ".b"].bfloat16(), stride=stride, padding=pad)

    x = px.bfloat16().contiguous(memory_format=torch.channels_last)
    x = F.relu(cv(x, "visual.conv1", 2, 1))
    x = F.relu(cv(x, "visual.conv2", 1, 1))
    x = F.avg_pool2d(F.relu(cv(x, "visual.conv3", 1, 1)), 2)
    for s, n in enumerate(a.layers):
        for j in range(n):
            p = "visual.layer%d.%d." % (s + 1, j)
            stride = 2 if (j == 0 and s > 0) else 1
            o = F.relu(cv(x, p + "conv1"))
            o = F.relu(cv(o, p + "conv2", 1, 1))
            if stride > 1:
                o = F.avg_pool2d(o, stride)
            o = cv(o, p + "conv3")
            idn = x
            if p + "downsample.0" in fw:
                idn = cv(F.avg_pool2d(x, stride) if stride > 1 else x, p + "downsample.0")
            x = F.relu(o + idn)
    at = "visual.attnpool."
    B, C = x.shape[:2]
    t = x.flatten(2).permute(0, 2, 1)
    t = torch.cat([t.float().mean(1, keepdim=True).bfloat16(), t], 1) + fw[at + "positional_embedding"]
    q = F.linear(t[:, :1], fw[at + "q_proj.weight"], fw[at + "q_proj.bias"].bfloat16())
    k = F.linear(t, fw[at + "k_proj.weight"], fw[at + "k_proj.bias"].bfloat16())
    v = F.linear(t, fw[at + "v_proj.weight"], fw[at + "v_proj.bias"].bfloat16())
    h = C // 64
    o = F.scaled_dot_product_attention(q.view(B, 1, h, 64).transpose(1, 2), k.view(B, -1, h, 64).transpose(1, 2),
                                       v.view(B, -1, h, 64).transpose(1, 2))
    f = F.linear(o.transpose(1, 2).reshape(B, C), fw[at + "c_proj.weight"], fw[at + "c_proj.bias"].bfloat16()).float()
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
    cls = {"conv3x3": 0.0, "gemm1x1": 0.0, "pools": 0.0, "attnpool": 0.0, "other": 0.0}
    for e in prof.key_averages():
        name = e.key
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        t /= 1e3
        if "conv3x3_bf16_wgmma_kernel" in name:
            cls["conv3x3"] += t
        elif "gemm_bf16_wgmma" in name:
            cls["gemm1x1"] += t
        elif "avgpool" in name or "stem_gather" in name or "attnpool_tokens" in name:
            cls["pools"] += t
        elif "attention" in name or "pool_proj" in name or "feat_norm" in name:
            cls["attnpool"] += t
        elif "Memcpy" not in name and "Memset" not in name:
            cls["other"] += t
    return cls


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
    for name in args.models.split(","):
        a = m.RESNET_ARCHS[name]
        sd = m.synthetic_state_dict(a, seed=0)
        model = m.B200Clip(a, device=0, max_batch=B).load_state_dict(sd)
        g = torch.Generator(device="cuda").manual_seed(0)
        px = torch.randn(B, 3, a.image_size, a.image_size, device="cuda", generator=g).clamp_(-1.8, 2.15)
        dt = _timed(lambda: model.embed_image_device(px), args.iters)
        gf = conv_gflop(a)
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
        fw = folded(sd, a)
        with torch.no_grad():
            dt_ref = _timed(lambda: cudnn_forward(fw, a, px), args.iters)
            ref = cudnn_forward(fw, a, px)
        cos = float((ours.float() * ref.float()).sum(-1).min())
        del fw
        torch.cuda.empty_cache()
        r = {"model": name, "images_per_s": B / dt, "gflop_per_image": gf, "tflops": gf * B / dt / 1e3,
             "split_ms": split, "batch1_ms_median": float(np.median(lat)), "cudnn_images_per_s": B / dt_ref,
             "min_cos_vs_cudnn": cos}
        out["models"].append(r)
        tot = sum(split.values()) or 1.0
        print("%-8s %8.0f img/s  %6.1f TFLOP/s (%.1f GFLOP/img)  conv3x3 %4.1f%%  1x1 %4.1f%%  pools %4.1f%%  attn+c_proj "
              "%4.1f%%  batch-1 %.2f ms  cuDNN %8.0f img/s  (min cos vs cuDNN %.4f)"
              % (name, r["images_per_s"], r["tflops"], gf, 100 * split["conv3x3"] / tot, 100 * split["gemm1x1"] / tot,
                 100 * split["pools"] / tot, 100 * split["attnpool"] / tot, r["batch1_ms_median"],
                 r["cudnn_images_per_s"], cos))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
