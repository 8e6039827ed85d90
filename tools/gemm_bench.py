#!/usr/bin/env python
"""Per-shape timing of the embed path's GEMM through b200_gemm_bf16_ex_device (CUDA events around one CUDA graph of
many launches, after warm-up).

  python tools/gemm_bench.py [--iters N] [--only SUBSTR] [--json OUT]

For each shape it times the column-block width forced to 128 (the 128 x 128 kernel) and to 256 (the persistent
128 x 256 kernel), and the library's automatic pick, with the epilogue the model uses on that GEMM (bias, quick-GELU
or erf-GELU on fc, residual in place on out-proj / c_proj, the patch-embedding row map).  It prints ms per launch,
TFLOP/s (2 M N K) and the fraction of the 989 TFLOP/s BF16 data-sheet rate, which kernel the automatic pick
launched, and, as a reference for what this card reaches on the shape, torch.matmul in bf16 (cuBLAS; not a code path
of the library).  Shapes: the eight ViT-L/14 layer GEMMs at batch 1024 and its patch embedding, the ViT-H/14 text
tower at batches 1, 8 and 64, and the ViT-B/32 image tower at batch 1024.  A width the library refuses prints "-".

  python tools/gemm_bench.py --ksweep [--json OUT]

splits the persistent kernel's time into k-loop and per-tile fixed cost: M = 1024 * 257 (ViT-L/14 image rows at batch
1024), N in {1024, 3072, 4096}, K in {256, 512, 1024, 2048, 4096}, bn forced to 256, for the plain (bias), quick-GELU
and in-place residual epilogues.  Per (N, flavour) it fits ms = waves * (a * k_blocks + b), waves = ceil(tiles / grid),
by least squares and prints a (us per 64-deep k-block), b (us per tile) and b / a (the fixed cost in k-blocks), with
the card's name, power limit and the SM clock sampled during each timed replay.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0   # H100 SXM data sheet, dense BF16


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in out.split(",")]


def tower_shapes(label, B, T, width, mlp, act):
    """(name, M, N, K, act, residual, group): qkv, out-proj (+ residual), fc (+ activation), c_proj (+ residual)."""
    M = B * T
    return [("%s qkv" % label, M, 3 * width, width, 0, False, 0),
            ("%s out" % label, M, width, width, 0, True, 0),
            ("%s fc" % label, M, mlp, width, act, False, 0),
            ("%s proj" % label, M, width, mlp, 0, True, 0)]


def shapes():
    out = tower_shapes("L/14 img b1024", 1024, 257, 1024, 4096, 1) + tower_shapes("L/14 txt b1024", 1024, 77, 768, 3072, 1)
    out.append(("L/14 patch b1024", 1024 * 256, 1024, 640, 0, True, 256))
    for B in (1, 8, 64):
        out += tower_shapes("H/14 txt b%d" % B, B, 77, 1024, 4096, 2)
    out += tower_shapes("B/32 img b1024", 1024, 50, 768, 3072, 1)
    return out


def sm_clock():
    return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]


def graph_ms(fn, iters, during=None):
    """ms per call of fn(stream) over one replay of a CUDA graph of `iters` calls (after warm-up); `during()` is called
    on the host while the timed replay runs."""
    import torch

    for _ in range(3):
        fn(torch.cuda.current_stream().cuda_stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = torch.cuda.current_stream().cuda_stream
        for _ in range(iters):
            fn(cap)
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    graph.replay()
    e1.record()
    if during is not None:
        during()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


KSWEEP_M = 1024 * 257
KSWEEP_N = (1024, 3072, 4096)
KSWEEP_K = (256, 512, 1024, 2048, 4096)
KSWEEP_FLAVOURS = (("plain", 0, False), ("quick-gelu", 1, False), ("residual", 0, True))


def ksweep(args, name, power):
    import numpy as np
    import torch
    from clip_retrieval_b200._lib import lib, check, GemmEpilogueC

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = KSWEEP_M
    t = {}   # (N, flavour, K) -> ms
    clocks = []
    for K in KSWEEP_K:
        g = torch.Generator(device="cuda").manual_seed(K)
        A = (torch.randn(M, K, device="cuda", generator=g, dtype=torch.bfloat16) * 0.5)
        for N in KSWEEP_N:
            W = (torch.randn(N, K, device="cuda", generator=g, dtype=torch.bfloat16) * K ** -0.5)
            bias = torch.randn(N, device="cuda", generator=g)
            out = torch.randn(M, N, device="cuda", generator=g, dtype=torch.bfloat16)
            for fl, act, res in KSWEEP_FLAVOURS:
                ep = GemmEpilogueC(bias.data_ptr(), out.data_ptr() if res else None, 0, 0, 0, 0, 0, act)

                def launch(s, ep=ep):
                    check(lib.b200_gemm_bf16_ex_device(A.data_ptr(), W.data_ptr(), out.data_ptr(), M, N, K, ep, 256, 0,
                                                       0, s), "gemm")

                est = graph_ms(launch, 2)
                # the timed replay lasts about 200 ms: the SM clock is sampled while it runs
                t[(N, fl, K)] = graph_ms(launch, max(3, min(500, int(200.0 / est))), lambda: clocks.append(sm_clock()))
                print("N=%-5d K=%-5d %-10s %8.4f ms  (SM clock %s)" % (N, K, fl, t[(N, fl, K)], clocks[-1]), flush=True)
            del W, bias, out
        del A
        torch.cuda.empty_cache()
    print("card: %s, power limit %s, SM clock sampled during the timings %s .. %s"
          % (name, power, min(clocks, key=lambda c: int(c.split()[0])), max(clocks, key=lambda c: int(c.split()[0]))))
    print("%-5s %-10s %12s %12s %10s" % ("N", "flavour", "a us/kblk", "b us/tile", "b/a kblk"))
    fits = []
    for N in KSWEEP_N:
        tiles = ((M + 127) // 128) * ((N + 255) // 256)
        waves = -(-tiles // min(tiles, sms))
        for fl, _, _ in KSWEEP_FLAVOURS:
            kblk = np.array([K / 64.0 for K in KSWEEP_K])
            y = np.array([t[(N, fl, K)] * 1e3 / waves for K in KSWEEP_K])   # us per wave
            a, b = np.polyfit(kblk, y, 1)
            fits.append({"N": N, "flavour": fl, "a_us_per_kblock": a, "b_us_per_tile": b, "b_over_a": b / a})
            print("%-5d %-10s %12.3f %12.3f %10.2f" % (N, fl, a, b, b / a))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": name, "power_limit": power, "sm_clocks": clocks, "M": M, "sms": sms,
                       "ms": [{"N": N, "flavour": fl, "K": K, "ms": v} for (N, fl, K), v in t.items()], "fits": fits},
                      f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", default=None, help="only shapes whose name contains this")
    ap.add_argument("--json", default=None)
    ap.add_argument("--ksweep", action="store_true", help="fit the persistent kernel's k-loop and per-tile costs")
    args = ap.parse_args()
    import torch
    import clip_retrieval_b200  # noqa: F401
    from clip_retrieval_b200._lib import lib, check, GemmEpilogueC

    if not torch.cuda.is_available():
        raise SystemExit("gemm_bench.py needs a CUDA device")
    name, power, clock = card()
    print("card: %s, power limit %s, max SM clock %s" % (name, power, clock))
    if args.ksweep:
        return ksweep(args, name, power)
    rows = []
    for sname, M, N, K, act, res, group in shapes():
        if args.only and args.only not in sname:
            continue
        g = torch.Generator(device="cuda").manual_seed(M + N + K)
        A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
        W = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).bfloat16()
        bias = torch.randn(N, device="cuda", generator=g)
        if group:
            # patch embedding: product row r -> output row (r / g) (g + 1) + 1 + r % g, positional row 1 + r % g
            out = torch.zeros(M // group * (group + 1), N, device="cuda", dtype=torch.bfloat16)
            pos = torch.randn(group + 1, N, device="cuda", generator=g).bfloat16()
            ep = GemmEpilogueC(None, pos.data_ptr(), 0, group, 1, 0, group, act)
        else:
            out = torch.randn(M, N, device="cuda", generator=g).bfloat16()
            ep = GemmEpilogueC(bias.data_ptr(), out.data_ptr() if res else None, 0, 0, 0, 0, 0, act)
        flops = 2.0 * M * N * K
        iters = args.iters if M >= 4096 else args.iters * 20

        def launch(bn, s):
            return lib.b200_gemm_bf16_ex_device(A.data_ptr(), W.data_ptr(), out.data_ptr(), M, N, K, ep, bn, 0, 0, s)

        def timed(fn):
            return graph_ms(fn, iters)

        r = {"shape": sname, "M": M, "N": N, "K": K}
        for label, bn in (("bn128", 128), ("bn256", 256), ("auto", 0)):
            if launch(bn, torch.cuda.current_stream().cuda_stream) != 0:
                r[label] = None
                continue
            torch.cuda.synchronize()
            r[label] = timed(lambda s, bn=bn: check(launch(bn, s), "gemm"))
        # which kernel the automatic pick launches
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            check(launch(0, torch.cuda.current_stream().cuda_stream), "gemm")
            torch.cuda.synchronize()
        kern = [e.name for e in prof.events() if "gemm_bf16" in e.name]
        r["auto_kernel"] = ("persistent 256" if "persistent" in kern[0] else "128-wide family") if kern else "?"
        Wt = W.t()
        r["cublas"] = timed(lambda s: torch.matmul(A, Wt))
        rows.append(r)

        def fmt(ms):
            if ms is None:
                return "%24s" % "-"
            tf = flops / (ms / 1e3) / 1e12
            return "%9.4f ms %6.1f TF %4.0f%%" % (ms, tf, 100 * tf / PEAK_TFLOPS)

        print("%-20s M=%-6d N=%-5d K=%-5d | bn128 %s | bn256 %s | auto %s (%s) | cuBLAS %s"
              % (sname, M, N, K, fmt(r["bn128"]), fmt(r["bn256"]), fmt(r["auto"]), r["auto_kernel"], fmt(r["cublas"])),
              flush=True)
        del A, W, bias, out
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": name, "power_limit": power, "max_sm_clock": clock, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
