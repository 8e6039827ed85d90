"""numpy restatement of OPQ training (b200_opq_train_f32, DESIGN.md §5 (xiii)).  TEST INFRASTRUCTURE.

FAISS OPQMatrix::train as recalled from its source (ASSUMED, FAISS cannot be run here), with this project's deliberate
differences:
  * initial rotation: the orthogonal polar factor of a seeded Gaussian d_out x d_in matrix (`gaussian`: Box-Muller on
    counter-based uniforms), instead of FAISS's float_randn(1234) followed by QR;
  * per iteration: xproj = X A^T; the PQ trained on xproj by this project's trainer (pq_train_ref.train_pq: niter_pq_0
    Lloyd iterations from the seeded picks at it = 0, then niter_pq iterations from the previous codebook, FAISS
    Train_hot_start); codes of the final codebook; Y = decode(codes); objective |xproj - Y|^2 / n; G = Y^T X;
    A = polar(G) = U V^T (orthogonal Procrustes), in float64.
`dtype` runs the float arithmetic of xproj, G and the SVD in float32 or float64; the PQ always sees fp32 rows.
"""
import numpy as np

import pq_train_ref as P

KSUB = P.KSUB


def _mix(x):
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def gaussian(d_out, d_in, seed):
    """Entry e: sqrt(-2 ln u1) cos(2 pi u2), u1 = ((h(2e) >> 11) + 1) 2^-53, u2 = (h(2e + 1) >> 11) 2^-53,
    h(c) = mix(seed ^ c * 0xD1342543DE82EF95)."""
    e = np.arange(d_out * d_in, dtype=np.uint64)
    with np.errstate(over="ignore"):
        a = _mix(np.uint64(seed) ^ ((np.uint64(2) * e) * np.uint64(0xD1342543DE82EF95)))
        b = _mix(np.uint64(seed) ^ ((np.uint64(2) * e + np.uint64(1)) * np.uint64(0xD1342543DE82EF95)))
    u1 = ((a >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0 ** -53
    u2 = (b >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return (np.sqrt(-2.0 * np.log(u1)) * np.cos(6.283185307179586 * u2)).reshape(d_out, d_in)


def polar(G, dtype=np.float64):
    """The orthogonal polar factor U V^T of G = U S V^T [d_out, d_in], d_out <= d_in."""
    U, _, Vt = np.linalg.svd(np.asarray(G, dtype), full_matrices=False)
    return U @ Vt


def initial_rotation(d_out, d_in, seed, dtype=np.float64):
    return polar(gaussian(d_out, d_in, seed), dtype)


def decode(codes, cb):
    M = cb.shape[0]
    return np.concatenate([cb[m][codes[:, m]] for m in range(M)], axis=1)


def pq_hot(X32, cb, niter):
    """pq_train_ref.train_pq's Lloyd iterations started from the codebook `cb` (FAISS Train_hot_start).
    Returns (codebook, sizes, codes of the final codebook, number of empty-codeword splits)."""
    X32 = np.asarray(X32, np.float32)
    n, d = X32.shape
    M, _, dsub = cb.shape
    X3 = X32.reshape(n, M, dsub)
    cb = np.array(cb, np.float32)
    eps = np.float32(1.0 / 1024.0)
    even = (np.arange(dsub) % 2) == 0
    splits = 0
    for it in range(niter + 1):
        codes = P.encode_codes(X32, cb)
        sizes = np.stack([np.bincount(codes[:, m], minlength=KSUB) for m in range(M)]).astype(np.int64)
        if it == niter:
            break
        S = np.zeros((M, KSUB, dsub), np.float32)
        order = np.argsort(codes, axis=0, kind="stable")
        start = np.concatenate([np.zeros((M, 1), np.int64), np.cumsum(sizes, axis=1)[:, :-1]], axis=1)
        mm, jj = np.nonzero(sizes)
        for p in range(int(sizes.max())):
            live = sizes[mm, jj] > p
            m_, j_ = mm[live], jj[live]
            S[m_, j_] = S[m_, j_] + X3[order[start[m_, j_] + p, m_], m_]
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
                splits += 1
    return cb, sizes, codes, splits


def train_opq(X, M, d_out=None, niter=50, niter_pq=4, niter_pq_0=40, seed=1234, dtype=np.float64, A0=None):
    """Returns (A [d_out, d_in] in `dtype`, objective [niter], total empty-codeword splits, the last codes / codebook)."""
    X = np.asarray(X, np.float32)
    n, d_in = X.shape
    d_out = d_in if d_out is None else d_out
    A = initial_rotation(d_out, d_in, seed, dtype) if A0 is None else np.asarray(A0, dtype)
    Xd = X.astype(dtype)
    obj, splits, cb, codes = [], 0, None, None
    for it in range(niter):
        xproj = Xd @ A.T.astype(dtype)
        xp32 = xproj.astype(np.float32)
        if it == 0:
            cb, _, codes = P.train_pq(xp32, M, niter_pq_0, seed)
            s = 0
        else:
            cb, _, codes, s = pq_hot(xp32, cb, niter_pq)
        splits += s
        Y = decode(codes, cb).astype(dtype)
        obj.append(float(((xproj - Y) ** 2).sum() / n))
        A = polar(Y.T @ Xd, dtype)
    return A, np.array(obj), splits, codes, cb


def procrustes_objective(A, G):
    """tr(A G^T): the quantity the polar factor of G maximises over matrices with orthonormal rows."""
    return float((np.asarray(A, np.float64) * np.asarray(G, np.float64)).sum())
