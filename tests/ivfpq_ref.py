"""CPU restatement of IVF-PQ search (8-bit codes, inner product).  TEST INFRASTRUCTURE.

FAISS IndexIVFPQ semantics for METRIC_INNER_PRODUCT, as restated in DESIGN.md §5 (viii) — ASSUMED from FAISS's
documentation and source layout, not observed (FAISS cannot be run here):
  * a query visits the `nprobe` lists whose fp32 centroids have the largest inner product with it (this engine finds
    them exactly; FAISS's HNSW coarse quantiser finds them approximately);
  * score of a row of list l with codes c: dis0(l) + sum_{m<M} T[m][c_m], where
        T[m][j] = sum_{t<dsub} q[m dsub + t] * codebook[m][j][t]   (one table per query),
        dis0(l) = q . centroid_l (fp32 centroids) when by_residual, else 0;
  * results by descending score, ties by ascending id; padding -1 / -FLT_MAX;
  * reconstruct(id) = codebook[m][c_m][t] + centroid_l[m dsub + t] in fp32 (no centroid without residuals);
  * a pre-transform maps queries to A q + b and reconstructions back by A^T (y - b).
"""
import numpy as np

from oracle import knn_ref

U32 = 2.0 ** -24   # unit roundoff of fp32


def gamma(n):
    """Higham's gamma_n = n u / (1 - n u): bound on the relative error of an n-term fp32 sum or dot product."""
    return n * U32 / (1 - n * U32)


def transform_f64(Q, A=None, b=None):
    """Queries as the index scores them, in float64: A q + b (or q without a transform)."""
    Q = np.asarray(Q, dtype=np.float32).astype(np.float64)
    if A is None:
        return Q
    out = Q @ np.asarray(A, np.float32).astype(np.float64).T
    return out if b is None else out + np.asarray(b, np.float32).astype(np.float64)


def tables_f64(Q64, codebook):
    """T [nq, M, 256] = per-subspace inner products of the queries with the codewords (float64)."""
    M, ksub, dsub = codebook.shape
    return np.einsum("qmt,mjt->qmj", Q64.reshape(Q64.shape[0], M, dsub), codebook.astype(np.float64))


def adc_scores_f64(Q64, centroids, codebook, codes, lists, by_residual):
    """Exact score [nq, n] of rows (codes [n, M], list [n]) for float64 queries (already pre-transformed)."""
    T = tables_f64(Q64, codebook)
    M = codebook.shape[0]
    S = np.zeros((Q64.shape[0], codes.shape[0]), dtype=np.float64)
    if by_residual:
        S += (Q64 @ centroids.astype(np.float64).T)[:, lists]
    for m in range(M):
        S += T[:, m, codes[:, m]]
    return S


def score_error_bound(Q64, centroids, codebook, codes, lists, by_residual, q_err=None):
    """Per (query, row) bound [nq, n] on |fp32 score - exact score|.

    dis0 is a d-term fp32 dot product: error <= gamma_d * sum_i |q_i c_i|.  A table entry is a dsub-term dot product:
    error <= gamma_dsub * sum_t |q_t cb_t|.  The score adds M + 1 terms (in any order): error <= gamma_{M+1} times
    the sum of their magnitudes (each at most its exact value plus its own bound).  `q_err` [nq, d] bounds the error
    of the fp32 pre-transformed query components, each of which perturbs the score by at most
    |q_err_i| * (|c_i| + |cb_i|)."""
    M, _, dsub = codebook.shape
    d = M * dsub
    Qa = np.abs(Q64)
    cba = np.abs(codebook.astype(np.float64))
    Ta = np.einsum("qmt,mjt->qmj", Qa.reshape(Qa.shape[0], M, dsub), cba)
    T = np.abs(tables_f64(Q64, codebook))
    terms = np.zeros((Q64.shape[0], codes.shape[0]))
    tab_err = np.zeros_like(terms)
    for m in range(M):
        terms += T[:, m, codes[:, m]] + gamma(dsub) * Ta[:, m, codes[:, m]]
        tab_err += gamma(dsub) * Ta[:, m, codes[:, m]]
    bound = tab_err
    if by_residual:
        ca = np.abs(centroids.astype(np.float64))
        d0a = (Qa @ ca.T)[:, lists]
        d0 = np.abs(Q64 @ centroids.astype(np.float64).T)[:, lists]
        bound = bound + gamma(d) * d0a
        terms += d0 + gamma(d) * d0a
    bound = bound + gamma(M + 1) * terms
    if q_err is not None:
        per = np.zeros((Q64.shape[0], codes.shape[0]))
        qe = np.abs(q_err).reshape(Q64.shape[0], M, dsub)
        for m in range(M):
            per += np.einsum("qt,nt->qn", qe[:, m], cba[m][codes[:, m]])
        if by_residual:
            per += (np.abs(q_err) @ np.abs(centroids.astype(np.float64)).T)[:, lists]
        bound = bound + per
    return bound


def pretransform_error_bound(Q, A, b=None):
    """Bound [nq, d] on |fp32 (A q + b) - exact|: a d_in-term dot product plus one add."""
    Qa = np.abs(np.asarray(Q, np.float32).astype(np.float64))
    Aa = np.abs(np.asarray(A, np.float32).astype(np.float64))
    s = Qa @ Aa.T
    if b is not None:
        s = s + np.abs(np.asarray(b, np.float32).astype(np.float64))
    return gamma(A.shape[1] + 1) * s


def ivfpq_search(Q32, centroids, codebook, codes, lists, k, nprobe, by_residual, ids=None):
    """fp32 restatement on already pre-transformed fp32 queries: exact float64 probes, then
    fp32(dis0) + T[0] + T[1] + ... added in m order in fp32; ties by ascending id.  Returns (D, I, probes)."""
    Q32 = np.asarray(Q32, np.float32)
    nq = Q32.shape[0]
    nlist = centroids.shape[0]
    M, _, dsub = codebook.shape
    ids = np.arange(codes.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, np.int64)
    Sc = Q32.astype(np.float64) @ centroids.astype(np.float64).T
    probes = np.argsort(-Sc, axis=1, kind="stable")[:, :min(nprobe, nlist)]
    T32 = np.einsum("qmt,mjt->qmj", Q32.reshape(nq, M, dsub), codebook.astype(np.float32)).astype(np.float32)
    D = np.full((nq, k), knn_ref.NEG, np.float32)
    I = np.full((nq, k), -1, np.int64)
    for q in range(nq):
        rows = np.nonzero(np.isin(lists, probes[q]))[0]
        if rows.size == 0:
            continue
        s = (Q32[q] @ centroids[lists[rows]].T).astype(np.float32) if by_residual else np.zeros(rows.size, np.float32)
        for m in range(M):
            s = (s + T32[q, m, codes[rows, m]]).astype(np.float32)
        d_, i_ = knn_ref.topk_from_scores(s[None], k, ids=ids[rows])
        D[q], I[q] = d_[0], i_[0]
    return D, I, probes


def reconstruct(centroids, codebook, codes, lists, by_residual):
    """Decoded rows [n, d] fp32: codeword + centroid with one fp32 add (codeword alone without residuals)."""
    M, _, dsub = codebook.shape
    y = codebook[np.arange(M)[None, :], codes.astype(np.int64)].reshape(codes.shape[0], M * dsub).astype(np.float32)
    if by_residual:
        y = (y + centroids[lists]).astype(np.float32)
    return y


def ivfpq_check(D, I, Q, centroids, codebook, codes, lists, k, nprobe, by_residual, A=None, b=None, id_base=0,
                probe_gap=1e-5, ids=None):
    """Verify an IVF-PQ result [nq, k] against float64 ADC scores of the rows of the float64 top-`nprobe` lists.

    Q are the queries as passed to the index (pre-transformed here in float64 when A is given).  Each query goes
    through knn_ref's tie-aware IVF check with its own tolerance: twice the largest score_error_bound over its
    candidates (the fp32 result and the float64 ranking may each sit anywhere inside that bound).  A query whose
    nprobe-th and (nprobe+1)-th float64 centroid scores are closer than `probe_gap` (plus the bound of the pre-transform
    error) may have been given another list by the fp32 coarse step; if it fails it is skipped.
    Returns (ok, message, n_checked)."""
    codes = np.asarray(codes)
    lists = np.asarray(lists, np.int64)
    ids = np.arange(codes.shape[0], dtype=np.int64) if ids is None else np.asarray(ids, np.int64)
    Q64 = transform_f64(Q, A, b)
    q_err = pretransform_error_bound(Q, A, b) if A is not None else None
    nq, nlist = Q64.shape[0], centroids.shape[0]
    nprobe = min(nprobe, nlist)
    Sc = Q64 @ centroids.astype(np.float64).T
    order = np.argsort(-Sc, axis=1, kind="stable")
    keep = np.ones(nq, dtype=bool)
    if nprobe < nlist:
        r = np.arange(nq)
        gap = probe_gap if q_err is None else probe_gap + 2 * (q_err @ np.abs(centroids.astype(np.float64)).max(axis=0))
        keep = Sc[r, order[:, nprobe - 1]] - Sc[r, order[:, nprobe]] >= gap
    checked = 0
    for q in range(nq):
        rows = np.nonzero(np.isin(lists, order[q, :nprobe]))[0]
        qe = None if q_err is None else q_err[q:q + 1]
        s = adc_scores_f64(Q64[q:q + 1], centroids, codebook, codes[rows], lists[rows], by_residual)[0]
        tol = 2 * score_error_bound(Q64[q:q + 1], centroids, codebook, codes[rows], lists[rows], by_residual, qe).max() \
            if rows.size else 0.0
        msg = knn_ref._ivf_check_one(D[q], I[q], s, ids[rows], k, id_base, tol)
        if msg is None:
            checked += 1
        elif keep[q]:
            return False, "query %d: %s" % (q, msg), checked
    return True, "ok", checked


# ---- fixtures: PQ training and encoding (numpy, CPU only; they exist to make realistic test indices) ----------
def train_pq(X, M, niter=4, seed=0):
    """Codebook [M, 256, d / M] by Lloyd iterations (squared L2) on each subspace of X [n, d]."""
    X = np.asarray(X, np.float32)
    n, d = X.shape
    dsub = d // M
    rng = np.random.default_rng(seed)
    cb = np.empty((M, 256, dsub), np.float32)
    for m in range(M):
        xs = X[:, m * dsub:(m + 1) * dsub]
        c = xs[rng.choice(n, 256, replace=n < 256)].copy()
        for _ in range(niter):
            a = encode_sub(xs, c)
            for j in np.unique(a):
                c[j] = xs[a == j].mean(axis=0)
        cb[m] = c
    return cb


def encode_sub(xs, c):
    """Index of the nearest codeword (squared L2, ties to the lower index) of every row of xs."""
    d2 = (xs.astype(np.float64) ** 2).sum(1)[:, None] - 2 * xs.astype(np.float64) @ c.astype(np.float64).T \
        + (c.astype(np.float64) ** 2).sum(1)[None, :]
    return np.argmin(d2, axis=1)


def encode(X, codebook):
    """Codes [n, M] uint8: nearest codeword of each subvector of X."""
    M, _, dsub = codebook.shape
    X = np.asarray(X, np.float32)
    return np.stack([encode_sub(X[:, m * dsub:(m + 1) * dsub], codebook[m]) for m in range(M)], axis=1).astype(np.uint8)


def make_index(n, d, nlist, M, seed=0, by_residual=True, niter=2):
    """A small realistic IVF-PQ index: unit centroids, rows = centroid + noise (normalised), lists by maximum inner
    product with the fp32 centroids, PQ trained on the residuals (or the rows).  Returns
    (centroids [nlist, d] f32, codebook, codes [n, M], lists [n], X [n, d] f32)."""
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    lists = rng.integers(0, nlist, n)
    X = C[lists] + 0.6 * rng.standard_normal((n, d)).astype(np.float32) / np.sqrt(d) * np.sqrt(d / 8.0)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    X = X.astype(np.float32)
    lists = np.argmax(X @ C.T, axis=1)
    R = X - C[lists] if by_residual else X
    cb = train_pq(R[: min(n, 8192)], M, niter=niter, seed=seed)
    codes = encode(R, cb)
    return C, cb, codes, lists.astype(np.int64), X
