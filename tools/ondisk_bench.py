"""On-disk IVF-PQ (populated.index + merged_index.ivfdata) served resident and streamed from host memory, on one GPU.

Setup per M: one quantiser trained with train_ivfpq on a sample of device-generated rows, `--parts` synthetic parts
encoded against it (index.encode) and written by faiss_io.write_ivfpq with their global ids in the lists, merged by
index_combiner into a folder under --dir (a temporary directory by default), the page cache warmed by one read of
merged_index.ivfdata.  Then for each (nprobe, nq, k): the same file loaded resident (max_device_bytes large) and
streamed (max_device_bytes=0), each timed over 20 / 5 / 2 host-entry searches (nq 1 / up to 64 / more) after one
warm-up, with

  qps          queries per wall second;
  staged_gbs   streamed: code bytes moved host -> device per wall second;
  gather / copy / scan   streamed: host gather time, device time of the host-to-device copies, list-scan kernel
               time, each as a share of the wall time of a search (they overlap, so they may add up past 1);
  same         streamed D and I equal the resident ones.

A pinned torch tensor of the largest staged byte count copied host -> device with cudaMemcpy (CUDA events) gives
the measured PCIe ceiling of this card in the same run.  Prints the card name and power limit first; one JSON line
per row, each also appended to --out as it is measured.

    python tools/ondisk_bench.py [--rows 20000000] [--M 64,128] [--dir /tmp/x] [--out results/ondisk.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in out.split(",")]


def build(m, folder, rows, d, nlist, M, parts, seed):
    import torch
    from clip_retrieval_b200 import faiss_io
    from clip_retrieval_b200.index import synth_rows

    spec = m.SynthSpec(seed=seed, clustered=True, nlist=nlist)
    sample = synth_rows(min(rows, 4 * nlist), d, spec, row0=0, dtype="float32")
    C, cb = m.train_ivfpq(sample, nlist, M, niter=4, pq_niter=8)
    del sample
    enc = m.B200IVFPQIndex(d, nlist, M, C, cb)
    src = os.path.join(folder, "parts")
    os.makedirs(src, exist_ok=True)
    bounds = np.linspace(0, rows, parts + 1).astype(np.int64)
    chunk = 1 << 20
    for i in range(parts):
        codes, lists = [], []
        for s in range(int(bounds[i]), int(bounds[i + 1]), chunk):
            e = min(int(bounds[i + 1]), s + chunk)
            c, l = enc.encode(synth_rows(e - s, d, spec, row0=s, dtype="float32"))
            codes.append(c.cpu().numpy())
            lists.append(l)
        torch.cuda.synchronize()
        faiss_io.write_ivfpq(os.path.join(src, "knn_%03d.index" % i), C, cb, np.concatenate(codes), np.concatenate(lists),
                             ids=np.arange(bounds[i], bounds[i + 1], dtype=np.int64), nprobe=16)
    out = os.path.join(folder, "merged")
    m.index_combiner(src, out)
    for f in os.listdir(src):
        os.remove(os.path.join(src, f))
    with open(os.path.join(out, "merged_index.ivfdata"), "rb") as f:   # warm the page cache
        while f.read(1 << 26):
            pass
    return out


def pinned_copy_gbs(nbytes):
    import torch

    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    g = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    g.copy_(h, non_blocking=True)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(5):
        g.copy_(h, non_blocking=True)
    b.record()
    torch.cuda.synchronize()
    return 5 * nbytes / (a.elapsed_time(b) * 1e-3) / 1e9


def timed(index, Q, k, reps):
    index.search(Q, k)
    t0 = time.perf_counter()
    for _ in range(reps):
        D, I = index.search(Q, k)
    return (time.perf_counter() - t0) / reps, D, I


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=20_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=65536)
    ap.add_argument("--M", default="64,128")
    ap.add_argument("--parts", type=int, default=4)
    ap.add_argument("--nprobe", default="16,64")
    ap.add_argument("--nq", default="1,64,1000")
    ap.add_argument("--k", default="40,3000")
    ap.add_argument("--dir", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--seed", type=int, default=1234)
    a = ap.parse_args()
    import torch
    import clip_retrieval_b200 as m

    name, power = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").close()

    def emit(r):
        print(json.dumps(r), flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(json.dumps(r) + "\n")

    emit({"card": name, "power_limit": power})
    top = a.dir or tempfile.mkdtemp(prefix="ondisk_bench_")
    for M in [int(x) for x in a.M.split(",")]:
        t0 = time.perf_counter()
        folder = build(m, os.path.join(top, "M%d" % M), a.rows, a.d, a.nlist, M, a.parts, a.seed)
        setup_s = time.perf_counter() - t0
        # the merged lists hold global ids out of list order: the resident index maps them (an id-mapped wrapper)
        res = m.load_index(folder, max_device_bytes=1 << 50)
        st = m.load_index(folder, max_device_bytes=0)
        res_in, st_in = getattr(res, "_index", res), getattr(st, "_index", st)
        rng = np.random.default_rng(a.seed)
        staged_max = 0
        for nprobe in [int(x) for x in a.nprobe.split(",")]:
            res_in.nprobe = st_in.nprobe = nprobe
            for nq in [int(x) for x in a.nq.split(",")]:
                Q = rng.standard_normal((nq, a.d)).astype(np.float32)
                Q /= np.linalg.norm(Q, axis=1, keepdims=True)
                for k in [int(x) for x in a.k.split(",")]:
                    reps = 20 if nq == 1 else (5 if nq <= 64 else 2)
                    tr, D0, I0 = timed(res, Q, k, reps)
                    ts, D1, I1 = timed(st, Q, k, reps)
                    s = st_in.last_stream_stats()
                    scan_ms, _ = st_in.last_scan_ms()
                    staged_max = max(staged_max, s["staged_bytes"])
                    r = {"card": name, "power_limit": power, "rows": a.rows, "nlist": a.nlist, "M": M,
                         "nprobe": nprobe, "nq": nq, "k": k, "setup_s": round(setup_s, 1),
                         "resident_qps": nq / tr, "streamed_qps": nq / ts, "streamed_ms": ts * 1e3,
                         "resident_ms": tr * 1e3, "staged_gbs": s["staged_bytes"] / ts / 1e9, "passes": s["passes"],
                         "gather": s["gather_ms"] / (ts * 1e3), "copy": s["copy_ms"] / (ts * 1e3),
                         "scan": scan_ms / (ts * 1e3),
                         "same": bool(np.array_equal(D0, D1) and np.array_equal(I0, I1))}
                    emit(r)
        ceiling = pinned_copy_gbs(max(staged_max, 1 << 20))
        r = {"card": name, "power_limit": power, "M": M, "pinned_h2d_gbs": ceiling, "bytes": staged_max}
        emit(r)
        del res, st, res_in, st_in
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
