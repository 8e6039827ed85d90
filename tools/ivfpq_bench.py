"""IVF-PQ search throughput on one GPU: a synthetic index (seeded centroids and codebook, random codes generated chunk by
chunk on the host from a seed and uploaded with add_codes), then one JSON line per (M, nprobe, nq, k) with the search
time, the list-scan kernel time, the code bytes and table lookups it implies, and the card it ran on.

    python tools/ivfpq_bench.py [--rows 200000000] [--nlist 65536] [--M 64,128,256] [--d 768]

The list scan reads M code bytes per probed row from HBM and does M random 4-byte table lookups in shared memory per
row; both rates are reported (against the 3.35 TB/s HBM3 data-sheet figure for the first).  Which one binds is read
from those two numbers, not assumed.  8 queries of every shape are checked against tests/ivfpq_ref.ivfpq_check on
their probed lists, with the codes regenerated on the host.  Rows are capped per M so that the code store and the
finalize copy fit in 80 GB (2 x rows x pitch <= 60 GB).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def gen_codes(seed, s, n, M):
    """Codes of rows [s, s + n): a deterministic function of (seed, chunk start)."""
    return np.random.default_rng([seed, s]).integers(0, 256, (n, M), dtype=np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000_000)
    ap.add_argument("--nlist", type=int, default=65536)
    ap.add_argument("--M", default="64,128,256")
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--nprobe", default="16,64")
    ap.add_argument("--nq", default="1,64,1000")
    ap.add_argument("--k", default="40,3000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1234)
    a = ap.parse_args()
    import torch
    import clip_retrieval_b200 as m
    import ivfpq_ref

    name, power = card()
    d, nlist = a.d, a.nlist
    rng = np.random.default_rng(a.seed)
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    Qall = rng.standard_normal((max(int(x) for x in a.nq.split(",")), d)).astype(np.float32)
    Qall /= np.linalg.norm(Qall, axis=1, keepdims=True)
    chunk = 1 << 24
    for M in (int(x) for x in a.M.split(",")):
        pitch = (M + 15) // 16 * 16
        n = min(a.rows, int(60e9 // (2 * pitch)))
        cb = (np.random.default_rng([a.seed, M]).standard_normal((M, 256, d // M)) * 0.05).astype(np.float32)
        lists_all = np.random.default_rng([a.seed, 7]).integers(0, nlist, n).astype(np.int32)
        idx = m.B200IVFPQIndex(d, nlist, M, C, cb)
        t0 = time.time()
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            idx.add_codes(gen_codes(a.seed, s, e - s, M), lists_all[s:e])
        idx.finalize()
        build_s = time.time() - t0
        sizes, _ = idx.invlists()
        # parity set: the rows of every list the 8 checked queries may probe, codes regenerated on the host
        nprobes = [int(x) for x in a.nprobe.split(",")]
        sel = np.arange(min(8, Qall.shape[0]))
        top = np.argsort(-(Qall[sel].astype(np.float64) @ C.T.astype(np.float64)), axis=1)[:, :max(nprobes) + 1]
        rows_ids = np.nonzero(np.isin(lists_all, np.unique(top)))[0]
        codes_sub = np.concatenate([gen_codes(a.seed, s, min(n, s + chunk) - s, M)[
            rows_ids[(rows_ids >= s) & (rows_ids < s + chunk)] - s] for s in range(0, n, chunk)])
        for nprobe in nprobes:
            idx.nprobe = nprobe
            probes_all = np.argsort(-(Qall.astype(np.float64) @ C.T.astype(np.float64)), axis=1)[:, :nprobe]
            for nq in (int(x) for x in a.nq.split(",")):
                Q = torch.from_numpy(Qall[:nq]).cuda()
                for k in (int(x) for x in a.k.split(",")):
                    for _ in range(2):   # warm-up: workspaces, attributes, graph capture at nq <= 4
                        idx.search_device(Q, k)
                    torch.cuda.synchronize()
                    times, scan = [], []
                    for _ in range(a.reps):
                        t = time.perf_counter()
                        D, I = idx.search_device(Q, k)
                        torch.cuda.synchronize()
                        times.append(time.perf_counter() - t)
                        scan.append(idx.last_scan_ms()[0] if nq > 4 else float("nan"))
                    ms = 1e3 * float(np.median(times))
                    rows_scanned = int(sizes[probes_all[:nq]].sum())
                    scan_ms = float(np.median(scan)) if nq > 4 else None
                    # parity: up to 8 queries against the oracle on their probed lists
                    qs = sel[:nq]
                    Dh, Ih = D.cpu().numpy()[qs], I.cpu().numpy()[qs]
                    ok, msg, nchk = ivfpq_ref.ivfpq_check(Dh, Ih, Qall[qs], C, cb, codes_sub, lists_all[rows_ids], k,
                                                          nprobe, True, ids=rows_ids)
                    rec = {"M": M, "rows": n, "nlist": nlist, "d": d, "nprobe": nprobe, "nq": nq, "k": k,
                           "ms": round(ms, 4), "qps": round(nq / (ms / 1e3), 1),
                           "scan_ms": None if scan_ms is None else round(scan_ms, 4),
                           "code_bytes_per_s_scan": None if scan_ms is None else rows_scanned * M / (scan_ms / 1e3),
                           "hbm_fraction_scan": None if scan_ms is None else rows_scanned * M / (scan_ms / 1e3) / HBM_BYTES_PER_S,
                           "lookups_per_s_scan": None if scan_ms is None else rows_scanned * M / (scan_ms / 1e3),
                           "rows_scanned": rows_scanned, "plan": list(idx.last_scan_plan()),
                           "parity": "ok" if ok else msg, "parity_checked": nchk, "build_s": round(build_s, 1),
                           "gpu": name, "power_limit": power}
                    print(json.dumps(rec), flush=True)
        del idx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
