"""IVF-PQ build throughput on one GPU: synthetic clustered rows generated on the device from a seed, then one JSON line
per M with the time of each stage (coarse k-means, PQ training, encoding), each between two device synchronisations,
and the card it ran on.

    python tools/ivfpq_build_bench.py [--rows 10000000] [--nlist 65536] [--M 64,128,256] [--d 768] [--train-rows 500000]

Encoding is two kernels per chunk.  The fused coarse assignment does 2 * n * nlist * d fp32 FMA flops; the codeword
step 3 * n * 256 * d (a subtraction and an fma per element and codeword).  Both are reported against the 67 TFLOP/s
FP32 data-sheet rate of the H100 SXM: the assignment is bound by FP32 FMA issue (its operands come from shared
memory, four 16-byte loads per 64 FMAs), so that is the bound its fraction names.  The coarse quantiser is trained on
the first `--train-rows` rows (`train_kmeans`), the PQ on the residuals of at most 65 536 of them (`train_ivfpq`).
8 rows of every shape are checked against tests/pq_train_ref.check_encode.

    python tools/ivfpq_build_bench.py --opq [--d 768] [--M 64] [--opq-niter 50]

`--opq` times OPQ training instead (`train_opq`, C ABI `b200_opq_train_f32`) on 65 536 anisotropic rows (a decaying
spectrum under a random rotation, made on the host from `--seed`): one JSON line per M with the training time split
into rotate (x A^T) / PQ (Lloyd iterations and the objective) / cross (G = Y^T X: 2 * n * d_in * d_out flops per
iteration, against the FP32 data-sheet rate) / SVD (fp64 cuSOLVER SVD and the polar product), each phase measured
between device synchronisations; the first and last objective; and the PQ error of the sample with and without the
rotation (plain PQ trained by `train_pq` with as many Lloyd iterations as OPQ ran in all).
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

FP32_FLOPS = 67e12   # H100 SXM data sheet, FP32 (non-tensor)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def opq_main(a):
    import torch
    import clip_retrieval_b200 as m

    name, power = card()
    n, d = m.index.PQ_TRAIN_MAX_ROWS, a.d
    rng = np.random.default_rng(a.seed)
    q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    X = torch.from_numpy(((rng.standard_normal((n, d)) * np.exp(-np.arange(d) / (d / 8))) @ q.T).astype(np.float32))
    X = X.cuda()
    Xn = X.cpu().numpy().astype(np.float64)

    def pq_error(rows, cb):
        M = cb.shape[0]
        codes, _ = m.B200IVFPQIndex(rows.shape[1], 1, M, np.zeros((1, rows.shape[1]), np.float32), cb,
                                    by_residual=False).encode(rows)
        codes = codes.cpu().numpy()
        Y = np.concatenate([cb[j][codes[:, j]] for j in range(M)], axis=1)
        return float(((rows.cpu().numpy().astype(np.float64) - Y) ** 2).sum() / rows.shape[0])

    for M in (int(x) for x in a.M.split(",")):
        m.train_opq(X[:4096], M, niter=1, niter_pq_0=1)       # warm-up: module load, cuSOLVER handle
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        A, obj, ph = m.train_opq(X, M, niter=a.opq_niter, seed=a.seed, phases=True)
        total = time.perf_counter() - t0
        lloyd = 40 + (a.opq_niter - 1) * 4
        cb, _ = m.train_pq(X, M, niter=lloyd, seed=a.seed)
        plain = pq_error(X, cb)
        Xr = m.index.pretransform_rows(X, A)
        cbr, _ = m.train_pq(Xr, M, niter=a.pq_niter, seed=a.seed)
        cross_flops = 2.0 * n * d * d * a.opq_niter
        rec = {"mode": "opq", "M": M, "rows": n, "d": d, "niter": a.opq_niter, "train_s": round(total, 3),
               "phase_ms": {k: round(v, 1) for k, v in ph.items()},
               "cross_flops_per_s": cross_flops / (ph["cross"] / 1e3) if ph["cross"] > 0 else None,
               "cross_fp32_datasheet_fraction": cross_flops / (ph["cross"] / 1e3) / FP32_FLOPS if ph["cross"] > 0 else None,
               "objective_first": float(obj[0]), "objective_last": float(obj[-1]),
               "pq_error_plain": plain, "pq_error_opq_codebook": float(obj[-1]),
               "pq_error_opq_retrained": pq_error(Xr, cbr), "plain_pq_lloyd_iterations": lloyd,
               "gpu": name, "power_limit": power}
        print(json.dumps(rec), flush=True)
        del Xr
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--nlist", type=int, default=65536)
    ap.add_argument("--M", default="64,128,256")
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--train-rows", type=int, default=500_000)
    ap.add_argument("--niter", type=int, default=10)
    ap.add_argument("--pq-niter", type=int, default=25)
    ap.add_argument("--chunk", type=int, default=1 << 20)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--opq", action="store_true", help="time OPQ training instead of the IVF-PQ build")
    ap.add_argument("--opq-niter", type=int, default=50)
    a = ap.parse_args()
    if a.opq:
        if a.M == ap.get_default("M"):
            a.M = "64"
        return opq_main(a)
    import torch
    import clip_retrieval_b200 as m
    import pq_train_ref as P

    name, power = card()
    d, nlist, n = a.d, a.nlist, a.rows
    spec = m.SynthSpec(seed=a.seed, clustered=True, centroid_seed=7, nlist=nlist)
    X = m.index.synth_rows(n, d, spec, dtype="float16")
    torch.cuda.synchronize()
    sel = np.linspace(0, n - 1, 8).astype(np.int64)
    Xs = X[torch.from_numpy(sel).cuda()].float().cpu().numpy()
    t0 = time.perf_counter()
    cent, _ = m.train_kmeans(X[:a.train_rows], nlist, niter=a.niter, seed=a.seed)   # shared by every M
    torch.cuda.synchronize()
    coarse_s = time.perf_counter() - t0
    for M in (int(x) for x in a.M.split(",")):
        t1 = time.perf_counter()
        # PQ training exactly as train_ivfpq does it, given the coarse centroids just trained
        ns = min(a.train_rows, m.index.PQ_TRAIN_MAX_ROWS)
        pick = torch.from_numpy(m.index.stride_picks(a.train_rows, ns, a.seed)).cuda()
        sample = X[pick].float().contiguous()
        tmp = m.B200IVFPQIndex(d, nlist, M, cent, np.zeros((M, 256, d // M), np.float32))
        res = torch.empty_like(sample)
        m._lib.check(m.lib.b200_index_encode_device(tmp._h, sample.data_ptr(), ns, None, res.data_ptr(), None,
                                                    torch.cuda.current_stream().cuda_stream), "encode")
        cb, _ = m.train_pq(res, M, niter=a.pq_niter, seed=a.seed)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        idx = m.B200IVFPQIndex(d, nlist, M, cent, cb)
        idx.encode(X[:a.chunk])          # warm-up: module load, first launches
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        codes, lists = idx.encode(X, chunk=a.chunk)
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        enc_s = t4 - t3
        ok, msg, _ = P.check_encode(codes[torch.from_numpy(sel).cuda()].cpu().numpy(), lists[sel], Xs, cent, cb, True)
        assign_flops = 2.0 * n * nlist * d
        code_flops = 3.0 * n * 256 * d
        rec = {"M": M, "rows": n, "nlist": nlist, "d": d, "train_rows": a.train_rows, "pq_train_rows": ns,
               "coarse_train_s": round(coarse_s, 2), "pq_train_s": round(t2 - t1, 2), "encode_s": round(enc_s, 2),
               "encode_rows_per_s": round(n / enc_s, 1),
               "encode_flops_per_s": (assign_flops + code_flops) / enc_s,
               "assign_flop_share": assign_flops / (assign_flops + code_flops),
               "fp32_datasheet_fraction": (assign_flops + code_flops) / enc_s / FP32_FLOPS,
               "bound": "fp32 FMA issue (coarse assignment)",
               "parity": "ok" if ok else msg, "gpu": name, "power_limit": power}
        print(json.dumps(rec), flush=True)
        del idx, tmp, codes
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
