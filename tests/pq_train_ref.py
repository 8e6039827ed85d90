"""CPU restatement of IVF-PQ encoding and PQ training (8-bit codes, inner-product coarse quantiser).  TEST INFRASTRUCTURE.

FAISS IndexIVFPQ semantics, as restated in DESIGN.md §5 (ix) — ASSUMED from FAISS's documentation and source layout,
not observed (FAISS cannot be run here):
  * coarse assignment: list(x) = argmax_l x' . c_l over the fp32 centroids, x' = A x + b with a pre-transform, ties to
    the lower list id;
  * residual r = x' - c_list in fp32 when by_residual, else x';
  * code_m = argmin_j sum_t (r[m dsub + t] - cb[m][j][t])^2, ties to the lower j.  The device computes each term as
    one rounded fp32 subtraction and one fma (the direct difference form, on purpose, not FAISS's expansion
    |r|^2 + |c|^2 - 2 r.c, which cancels for residuals close to a codeword);
  * PQ training: M independent Lloyd k-means of 256 codewords (squared L2), initial codewords one seeded pick per
    stride of the rows (oracle.kmeans_ref.initial_picks, the same picks for every m), codeword = the fp32 sum of its
    rows in ascending row order times fp32 1/count, an empty codeword takes a perturbed copy of the largest one of the
    same m (ties to the lower id; 1 +- 1/1024 alternating by column; sizes halve).
"""
import numpy as np

from oracle.kmeans_ref import initial_picks

import ivfpq_ref

U32 = ivfpq_ref.U32
gamma = ivfpq_ref.gamma
KSUB = 256
MAX_TRAIN = 65536


def sample_picks(n, count, seed):
    """Rows of the PQ training sample: one seeded pick per stride (all rows when n <= count)."""
    return initial_picks(n, min(n, count), seed)


def coarse_scores_f64(X, C):
    """[n, nlist] float64 inner products of (already pre-transformed) rows with the centroids."""
    return np.asarray(X, np.float64) @ np.asarray(C, np.float32).astype(np.float64).T


def coarse_assign(X, C):
    """argmax over the float64 scores, ties to the lower list id.  On data where every fp32 product and sum is exact
    the device's fp32 argmax is this one bit for bit."""
    return np.argmax(coarse_scores_f64(X, C), axis=1)


def residuals(X32, C, lists, by_residual):
    """fp32 residuals x' - c_list (one fp32 subtraction per element), or x' itself."""
    X32 = np.asarray(X32, np.float32)
    return (X32 - np.asarray(C, np.float32)[lists]).astype(np.float32) if by_residual else X32.copy()


def sub_distances_f64(R, cb):
    """[n, M, 256] float64 squared distances of each fp32 residual sub-vector to each codeword."""
    M, _, dsub = cb.shape
    R3 = np.asarray(R, np.float64).reshape(R.shape[0], M, 1, dsub)
    out = np.empty((R.shape[0], M, KSUB))
    for m in range(M):
        out[:, m] = ((R3[:, m] - cb[m].astype(np.float64)[None]) ** 2).sum(-1)
    return out


def encode_codes(R, cb):
    """codes [n, M] uint8: argmin over the float64 distances, ties to the lower codeword."""
    return np.argmin(sub_distances_f64(R, cb), axis=2).astype(np.uint8)


def encode(X32, C, cb, by_residual):
    """(codes, lists) of (already pre-transformed) fp32 rows."""
    lists = coarse_assign(X32, C)
    return encode_codes(residuals(X32, C, lists, by_residual), cb), lists


def list_error_bound(X64, C, x_err=None):
    """[n, nlist] bound on |fp32 score - exact score| of x . c_l.

    A d-term fp32 dot product (fma chain in any order): |err| <= gamma_d * sum_i |x_i c_i| (Higham 3.1).  When the
    rows themselves carry an error |x_err_i| (fp32 pre-transform against the exact A x + b), the exact score moves by
    at most sum_i |x_err_i| |c_i| more."""
    Ca = np.abs(np.asarray(C, np.float32).astype(np.float64))
    b = gamma(C.shape[1]) * (np.abs(X64) @ Ca.T)
    if x_err is not None:
        b = b + np.abs(x_err) @ Ca.T
    return b


def codeword_error_bound(R64, cb, r_err=None):
    """[n, M, 256] bound on |fp32 distance - exact distance| of sub-vector m of r to codeword j.

    Each term: e_t = fl(r_t - c_t) = (r_t - c_t)(1 + d_t), |d_t| <= u, so e_t^2 = (r_t - c_t)^2 (1 + 2u + u^2) at worst;
    the dsub-term fp32 sum of the e_t^2 (fma: e_t * e_t + s rounded once) adds gamma_dsub relative to the sum of its
    non-negative terms.  Together: |err| <= gamma_{dsub + 2} * sum_t (r_t - c_t)^2, since (1 + gamma_dsub)(1 + u)^2
    <= 1 + gamma_{dsub + 2}.  When the residual components are only known to within |r_err_t| of r (pre-transform),
    the exact distance moves by at most sum_t (2 |r_t - c_t| |r_err_t| + r_err_t^2) more."""
    M, _, dsub = cb.shape
    D = sub_distances_f64(R64, cb)
    b = gamma(dsub + 2) * D
    if r_err is not None:
        E = np.abs(np.asarray(r_err, np.float64)).reshape(R64.shape[0], M, 1, dsub)
        R3 = np.asarray(R64, np.float64).reshape(R64.shape[0], M, 1, dsub)
        for m in range(M):
            diff = np.abs(R3[:, m] - cb[m].astype(np.float64)[None])
            b[:, m] += (2 * diff * E[:, m] + E[:, m] ** 2).sum(-1) * (1 + 4 * U32)
    return b


def train_pq(X32, M, niter, seed=1234):
    """Restatement of b200_pq_train_f32.  Returns (codebook float32 [M, 256, dsub], sizes int64 [M, 256], codes of the
    final codebook).  Assignment by float64 argmin (the device's fp32 argmin whenever the top-2 gap exceeds the bound);
    sums in fp32, row after row in ascending row order."""
    X32 = np.asarray(X32, np.float32)
    n, d = X32.shape
    dsub = d // M
    X3 = X32.reshape(n, M, dsub)
    cb = np.ascontiguousarray(X3[initial_picks(n, KSUB, seed)].transpose(1, 0, 2))   # [M, 256, dsub]
    eps = np.float32(1.0 / 1024.0)
    even = (np.arange(dsub) % 2) == 0
    codes = None
    sizes = None
    for it in range(niter + 1):
        codes = encode_codes(X32, cb)
        sizes = np.stack([np.bincount(codes[:, m], minlength=KSUB) for m in range(M)]).astype(np.int64)
        if it == niter:
            break
        # fp32 sums in ascending row order, all (m, j) buckets at once: step p adds the p-th row of every bucket
        S = np.zeros((M, KSUB, dsub), np.float32)
        order = np.argsort(codes, axis=0, kind="stable")          # [n, M]: rows of each m sorted by code, stable
        start = np.concatenate([np.zeros((M, 1), np.int64), np.cumsum(sizes, axis=1)[:, :-1]], axis=1)
        mm, jj = np.nonzero(sizes)
        for p in range(int(sizes.max())):
            live = sizes[mm, jj] > p
            m_, j_ = mm[live], jj[live]
            rows = order[start[m_, j_] + p, m_]
            S[m_, j_] = S[m_, j_] + X3[rows, m_]
        inv = (np.float32(1.0) / np.maximum(sizes, 1).astype(np.float32)).astype(np.float32)
        upd = sizes > 0
        cb[upd] = S[upd] * inv[upd][:, None]
        for m in range(M):
            sz = sizes[m].copy()
            for ci in range(KSUB):
                if sz[ci] != 0:
                    continue
                cj = int(np.argmax(sz))
                if sz[cj] < 2:
                    break
                v = cb[m, cj].copy()
                cb[m, ci] = np.where(even, v * (np.float32(1) + eps), v * (np.float32(1) - eps))
                cb[m, cj] = np.where(even, v * (np.float32(1) - eps), v * (np.float32(1) + eps))
                sz[ci] = sz[cj] // 2
                sz[cj] -= sz[ci]
    return cb, sizes, codes


def codeword_gaps(R, cb):
    """Per (row, m): float64 distance gap between the nearest and the second-nearest codeword, and the bound of the
    two (the device's fp32 argmin is the float64 one whenever the gap exceeds the bound)."""
    D = sub_distances_f64(R, cb)
    part = np.partition(D, 1, axis=2)
    return part[..., 1] - part[..., 0], gamma(cb.shape[2] + 2) * (part[..., 1] + part[..., 0])


def check_encode(codes, lists, X32, C, cb, by_residual, x_err=None):
    """Tolerant check of device (codes, lists) for fp32 rows X32 (already pre-transformed in float64 / fp32, with
    `x_err` bounding each component's error).  A chosen list must score within the bound of the best one; the chosen
    codeword (on the residual of the chosen list) within the bound of the nearest one.  Returns
    (ok, message, rows decided inside a bound)."""
    X64 = np.asarray(X32, np.float64)
    lists = np.asarray(lists, np.int64)
    S = coarse_scores_f64(X64, C)
    B = list_error_bound(X64, C, x_err)
    r = np.arange(X64.shape[0])
    best = np.argmax(S, axis=1)
    slack = B[r, lists] + B[r, best]
    bad = S[r, lists] < S[r, best] - slack
    if bad.any():
        i = int(np.nonzero(bad)[0][0])
        return False, "row %d: list %d scores %.9g, best %d scores %.9g (bound %.3g)" % (
            i, lists[i], S[i, lists[i]], best[i], S[i, best[i]], slack[i]), 0
    close_list = (S[r, best] - np.partition(S, -2, axis=1)[:, -2] <= slack) if C.shape[0] > 1 else np.zeros(len(r), bool)
    if by_residual:
        R64 = X64 - np.asarray(C, np.float32).astype(np.float64)[lists]
        r_err = None if x_err is None else np.abs(x_err) + U32 * np.abs(R64)
        if x_err is None:   # the device's fp32 residual is exact here: recompute it as the device does
            R64 = residuals(np.asarray(X32, np.float32), C, lists, True).astype(np.float64)
    else:
        R64, r_err = X64, x_err
    D = sub_distances_f64(R64, cb)
    Bc = codeword_error_bound(R64, cb, r_err)
    M = cb.shape[0]
    mm = np.arange(M)[None, :]
    c = np.asarray(codes, np.int64)
    near = np.argmin(D, axis=2)
    slack = Bc[r[:, None], mm, c] + Bc[r[:, None], mm, near]
    bad = D[r[:, None], mm, c] > D[r[:, None], mm, near] + slack
    if bad.any():
        i, m = (int(v) for v in np.argwhere(bad)[0])
        return False, "row %d m %d: code %d distance %.9g, nearest %d %.9g (bound %.3g)" % (
            i, m, c[i, m], D[i, m, c[i, m]], near[i, m], D[i, m, near[i, m]], slack[i, m]), 0
    part = np.partition(D, 1, axis=2)
    close_code = (part[..., 1] - part[..., 0] <= 2 * gamma(cb.shape[2] + 2) * part[..., 1] + (
        0 if r_err is None else Bc.max(axis=2))).any(axis=1)
    return True, "ok", int((close_list | close_code).sum())
