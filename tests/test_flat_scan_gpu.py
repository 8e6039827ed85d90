"""Flat exhaustive scan against float64, kernel by kernel (csrc/knn_scan.cu, csrc/knn_mma.cu).

Every case of tests/flat_scan_cases.py runs here and asserts the plan the library reports for it
(`last_scan_plan()`: kernel, queries per pass, chunks per lane), so each of the 11 ring, 17 register and 8 range
instantiations is proven to have run.  Results are checked with knn_ref.check_topk against float64 scores of rows
regenerated on the host (oracle/synth_ref), never read back through the index under test; reconstructed rows
must equal the stored fp16 rows bit for bit.  Beyond the instantiations: both sides of every dispatch switch,
k at the warp-list edges and the 8192 maximum, stores smaller than one 32-row slot or than the grid, exact ties
across warps, slots and CTAs (and through the k-th boundary), all-zero queries, NaN rows on every path, range
search at every width with FAISS's strict `>` pinned exactly, and the shard merge at its 16384-candidate limit.
"""
import functools

import numpy as np
import pytest

from oracle import knn_ref, synth_ref
from flat_scan_cases import (BOUNDARY_CASES, DEFAULT, FMA_REGISTER, FMA_RING, HI_ONLY, INSTANTIATION_CASES, K_CASES,
                             RANGE_WIDTHS, REGISTER, SPLIT, STAGED, WIDTHS, ch_of)

pytestmark = pytest.mark.gpu
TOL = 2e-6
SEED = 1234
CHUNK = 16384
N = 38021   # 9 slots of 32 rows per CTA of the ring (more than its 8 stages) + a partial slot and a partial 4-row block


@functools.lru_cache(maxsize=2)
def _rows(n, d):
    """Synthetic rows 0..n-1 regenerated on the host in chunks (bounded temporaries).  Read-only: copy to edit."""
    X = np.concatenate([synth_ref.rows_f16(min(CHUNK, n - s), d, row0=s, seed=SEED) for s in range(0, n, CHUNK)])
    X.flags.writeable = False
    return X


def _queries(nq, d, X=None, seed=4321):
    """Unit queries; with X, query 0 is the last stored row (so the last, partial slot holds the best match)."""
    Q = synth_ref.rows_f32(nq, d, seed=seed)
    if X is not None:
        Q[0] = X[-1].astype(np.float32)
    return Q


def _index(d, n=None, X=None, flags=DEFAULT):
    import clip_retrieval_b200 as m

    idx = m.B200FlatIndex(d)
    if X is None:
        idx.add_synthetic(n, m.SynthSpec(seed=SEED))
    else:
        idx.add(X)
    idx.set_tensor_scan(flags)
    return idx


def _plan(idx, expect, what):
    plan = idx.last_scan_plan()
    assert plan[:3] == tuple(expect), "%s: ran (kernel, NQ, CH) = %r, expected %r" % (what, plan[:3], tuple(expect))
    assert (plan[3] > 0) == (plan[0] != REGISTER), "%s: ring stages %d for kernel %d" % (what, plan[3], plan[0])


def _check_rows(R, I, X, what):
    """Reconstructed rows: the stored fp16 row upcast, bit for bit; NaN where the id is -1."""
    m = I >= 0
    assert np.array_equal(R[m].view(np.uint32), X[I[m]].astype(np.float32).view(np.uint32)), "%s: rows differ" % what
    assert np.isnan(R[~m]).all(), "%s: padding rows are not NaN" % what


def _search(idx, X, Q, k, what, expect=None, reconstruct=True, S64=None, ids=None):
    """Host search (never a graph replay), plan check, then check_topk against float64 over the candidate `ids`."""
    if reconstruct:
        D, I, R = idx.search_and_reconstruct(Q, k)
        _check_rows(R, I, X, what)
    else:
        D, I = idx.search(Q, k)
    if expect is not None:
        _plan(idx, expect, what)
    if S64 is None:
        S64 = knn_ref.scores_f64(X, Q)
    if ids is not None:
        S64 = S64[:, ids]
    ok, msg, _ = knn_ref.check_topk(D, I, S64, k, ids=ids, tol=TOL)
    assert ok, "%s: %s" % (what, msg)
    return D, I


def _agree(I1, I2, S64, what, limit=None):
    """Two searches of the same queries return the same ids, except where swapped ids' float64 scores are within
    2 * TOL.  `limit`: ids >= limit exist in only one of the two stores and are dropped before comparing."""
    for q in range(I1.shape[0]):
        a, b = I1[q], I2[q]
        if limit is not None:
            a, b = a[a < limit], b[b < limit]
            a, b = a[:min(a.size, b.size)], b[:min(a.size, b.size)]
        for j in np.nonzero(a != b)[0]:
            assert a[j] >= 0 and b[j] >= 0 and abs(S64[q, a[j]] - S64[q, b[j]]) <= 2 * TOL, (
                "%s: query %d rank %d holds id %d on one side and %d on the other" % (what, q, j, a[j], b[j]))


def _device_twice(idx, Q, k):
    """search_device with reconstruction twice: the first call of a shape runs eagerly, the second replays the CUDA
    graph captured for it."""
    import torch

    t = torch.from_numpy(np.ascontiguousarray(Q)).cuda()
    return [[o.cpu().numpy() for o in idx.search_device(t, k, reconstruct=True)] for _ in range(2)]


# ---- every instantiation --------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("d", WIDTHS)
def test_every_instantiation(d):
    """Each (kernel, NQ, CH) at a width ending inside its last chunk and at the full width, with the last pass of
    NQ = 2 and NQ = 4 partly empty; serving shapes (nq <= 4) also through search_device, eagerly and then from the
    captured CUDA graph, which must reproduce the host search bit for bit."""
    k = 40
    X = _rows(N, d)
    idx = _index(d, N)
    for dd, nq, flags, expect in INSTANTIATION_CASES:
        if dd != d:
            continue
        what = "d %d nq %d flags %d" % (d, nq, flags)
        idx.set_tensor_scan(flags)
        Q = _queries(nq, d, X)
        D, I = _search(idx, X, Q, k, what, expect)
        assert I[0, 0] == N - 1, "%s: the last row, equal to query 0, is not its best match: %r" % (what, I[0, :4])
        if nq <= 4:
            (De, Ie, Re), (Dg, Ig, Rg) = _device_twice(idx, Q, k)
            assert np.array_equal(Ie, I) and np.array_equal(De, D), what + ": eager search_device differs from search"
            assert np.array_equal(Ig, Ie) and np.array_equal(Dg, De), what + ": graph replay differs from eager"
            assert np.array_equal(Rg.view(np.uint32), Re.view(np.uint32)), what + ": graph replay rows differ"
            _check_rows(Re, Ie, X, what)
            _plan(idx, expect, what + " (after the graph replay)")


# ---- dispatch boundaries --------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", sorted(BOUNDARY_CASES))
def test_dispatch_boundaries(name):
    """Both sides of each switch of the dispatch: the tensor scan (nq > 4, k <= 128, n >= 4096, d >= 64), the
    halving of queries per pass at NQ * k > 1536, the ring-to-register fallback, and the 64-query batches of the
    FMA path.  Each side runs the kernel it must, matches float64, and returns the ids of the other side."""
    cases = BOUNDARY_CASES[name]
    d = cases[0][0]
    nmax = max(c[3] for c in cases)
    X = _rows(nmax, d)
    Q = _queries(max(c[1] for c in cases), d)
    S64 = knn_ref.scores_f64(X, Q)
    idxs = {}
    got = []
    for dd, nq, k, n, flags, expect in cases:
        if n not in idxs:
            idxs[n] = _index(d, n)
        idx = idxs[n]
        idx.set_tensor_scan(flags)
        what = "%s: nq %d k %d n %d flags %d" % (name, nq, k, n, flags)
        D, I = _search(idx, X[:n], Q[:nq], k, what, expect, reconstruct=nq * k * d <= (1 << 24), S64=S64[:nq, :n])
        if expect[0] == HI_ONLY:
            assert idx.last_hi_only_fallbacks() == 0, what + ": iid rows, yet a hi-only proof failed"
        got.append((nq, k, n, I))
    for nq1, k1, n1, I1 in got:
        for nq2, k2, n2, I2 in got:
            q, kk = min(nq1, nq2), min(k1, k2)
            _agree(I1[:q, :kk], I2[:q, :kk], S64, "%s: n %d/%d" % (name, n1, n2), limit=min(n1, n2) if n1 != n2 else None)


# ---- k range ----------------------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("d,flags", [(200, FMA_REGISTER), (1288, FMA_REGISTER), (200, DEFAULT), (776, DEFAULT)],
                         ids=["register-d200", "register-d1288", "ring-d200", "ring-d776"])
def test_k_range(d, flags):
    """k = 1, the warp-list edges 31/32/33 and the 8192 maximum at nq 1, 2 and 4; k = 8193 is refused with the
    documented error before any CUDA work."""
    import torch
    from clip_retrieval_b200 import _lib

    n = 20011
    X = _rows(n, d)
    idx = _index(d, n, flags=flags)
    Q = _queries(4, d, X)
    S64 = knn_ref.scores_f64(X, Q)
    for dd, nq, k, fl, expect in K_CASES:
        if (dd, fl) != (d, flags):
            continue
        _search(idx, X, Q[:nq], k, "d %d nq %d k %d flags %d" % (d, nq, k, flags), expect, reconstruct=k < 8192,
                S64=S64[:nq])
    launches = _lib.launch_count()
    for call in (lambda: idx.search(Q, 8193), lambda: idx.search_and_reconstruct(Q, 8193),
                 lambda: idx.search_device(torch.from_numpy(Q).cuda(), 8193)):
        with pytest.raises(ValueError, match="exceeds the supported maximum of 8192"):
            call()
    assert _lib.launch_count() == launches


@pytest.mark.timeout(300)
@pytest.mark.parametrize("flags,kernel", [(DEFAULT, STAGED), (FMA_REGISTER, REGISTER)], ids=["ring", "register"])
def test_k_at_least_n_returns_every_row(flags, kernel):
    """k >= n: every row comes back in float64 order, negative scores included (the ordered-key mapping of
    negative floats), then -1 / -FLT_MAX."""
    d, n, k = 200, 100, 128
    X = _rows(n, d)
    idx = _index(d, n, flags=flags)
    Q = _queries(3, d)
    S64 = knn_ref.scores_f64(X, Q)
    D, I = _search(idx, X, Q, k, "k >= n", (kernel, 2, 1), S64=S64)
    assert (D[:, :n] < 0).sum(axis=1).min() > 20          # plenty of negative scores in every query
    want = np.stack([np.lexsort((np.arange(n), -S64[q])) for q in range(3)])
    assert np.array_equal(I[:, :n], want)
    assert (I[:, n:] == -1).all() and (D[:, n:] == knn_ref.NEG).all()


# ---- small and sparse stores ----------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("flags,kernel", [(FMA_RING, STAGED), (FMA_REGISTER, REGISTER)], ids=["ring", "register"])
def test_small_and_sparse_stores(flags, kernel):
    """Stores smaller than one 4-row block, one 32-row slot, and (3200 rows = 100 slots) than the grid, so most
    warps' lists stay empty: every row found, -1 / -FLT_MAX padding past them, for NQ = 1, 2 and 4."""
    d = 264
    for n in (1, 3, 4, 5, 31, 32, 33, 3200):
        X = _rows(n, d)
        idx = _index(d, n, flags=flags)
        for nq, NQ in ((1, 1), (3, 2), (7, 4)):
            Q = _queries(nq, d, X)
            for k in (5, 40):
                _search(idx, X, Q, k, "n %d nq %d k %d" % (n, nq, k), (kernel, NQ, ch_of(d)))


# ---- ties and all-zero queries --------------------------------------------------------------------------------

TIE_IDS = np.array([3, 6, 7, 33, 70, 4100, 17000, N - 1])   # 4-row blocks 0 and 1 (twice), other slots, other CTAs


def _tie_paths():
    """(flags, nq, expected plan, which queries hold the tied row, which are all zero) per path."""
    return [
        (DEFAULT, 3, (STAGED, 2, 1), [0, 2], [1]),
        (FMA_REGISTER, 3, (REGISTER, 2, 1), [0, 2], [1]),
        (FMA_RING, 7, (STAGED, 4, 1), [0, 3, 6], [1, 5]),
        (FMA_REGISTER, 7, (REGISTER, 4, 1), [0, 3, 6], [1, 5]),
        (DEFAULT, 64, (SPLIT, 128, 1), [0, 17, 63], [1, 40]),
        (DEFAULT, 200, (HI_ONLY, 256, 1), [0, 130, 199], [1, 129]),
    ]


@pytest.mark.timeout(300)
def test_ties_across_warps_slots_and_ctas():
    """Copies of one row at ids in different 4-row blocks, 32-row slots and CTAs: a query equal to the row gets them
    first, in ascending id order, and a k smaller than the group returns its lowest ids.  An all-zero query scores
    every row exactly 0 and must get ids 0..k-1.  On the ring, register, split and hi-only paths."""
    d = 256
    X = _rows(N, d).copy()
    X[TIE_IDS] = X[TIE_IDS[0]]
    idx = _index(d, X=X)
    r = X[TIE_IDS[0]].astype(np.float32)
    for flags, nq, expect, tied, zero in _tie_paths():
        Q = _queries(nq, d)
        Q[tied] = r
        Q[zero] = 0.0
        S64 = knn_ref.scores_f64(X, Q)
        idx.set_tensor_scan(flags)
        for k in (1, 5, 8, 40):
            what = "flags %d nq %d k %d" % (flags, nq, k)
            D, I = _search(idx, X, Q, k, what, expect, reconstruct=nq <= 7, S64=S64)
            c = min(k, TIE_IDS.size)
            for q in tied:
                assert np.array_equal(I[q, :c], TIE_IDS[:c]), "%s: query %d: %r" % (what, q, I[q, :c])
                assert (D[q, :c] == D[q, 0]).all(), what
            for q in zero:
                assert np.array_equal(I[q], np.arange(k)) and (D[q] == 0).all(), "%s: zero query %d: %r" % (what, q, I[q])
            if expect[0] == HI_ONLY:
                assert idx.last_hi_only_fallbacks() >= len(zero), what + ": a zero query passed the hi-only proof"


# ---- NaN rows ---------------------------------------------------------------------------------------------------

def _with_nan_rows(X, all_nan, one_nan):
    """X with rows `all_nan` entirely NaN and rows `one_nan` (id -> column) holding one NaN; returns X, finite ids."""
    X = X.copy()
    X[all_nan] = np.float16(np.nan)
    for i, c in one_nan.items():
        X[i, c] = np.float16(np.nan)
    finite = np.nonzero(~np.isnan(X).any(axis=1))[0]
    return X, finite


def _nan_paths(d):
    ch = ch_of(d)
    return [(DEFAULT, 3, (STAGED, 2, ch)), (FMA_REGISTER, 3, (REGISTER, 2, ch)), (FMA_RING, 7, (STAGED, 4, ch)),
            (FMA_REGISTER, 7, (REGISTER, 4, ch)), (DEFAULT, 64, (SPLIT, 128, ch)), (DEFAULT, 200, (HI_ONLY, 256, ch))]


@pytest.mark.timeout(300)
def test_nan_rows_are_never_returned():
    """Rows entirely NaN (id 0, in a 4-row block, the last row) and rows with one NaN (first column, last column of a
    partial chunk, middle): never returned, their neighbours' results unchanged, on every path.  A NaN row makes
    the hi-only error bound infinite, so every query of that batch must fail its proof and be re-run in split
    mode, including an all-zero query whose bound is 0 * inf = NaN."""
    d, k = 520, 40
    X, finite = _with_nan_rows(_rows(N, d), [0, 4101, N - 1], {5: 0, 6: d - 1, 2000: 300})
    idx = _index(d, X=X)
    for flags, nq, expect in _nan_paths(d):
        Q = _queries(nq, d)
        # neighbours of the NaN rows, scaled (exactly) to scores near 0.25: at a score of 1 the fp32 accumulation of
        # the wgmma scan alone reaches TOL (2.06e-6 observed for a self-match at d = 520)
        Q[:3] = 0.25 * X[[1, 4, N - 2]].astype(np.float32)
        if nq > 3:
            Q[3] = 0.0
        idx.set_tensor_scan(flags)
        what = "flags %d nq %d" % (flags, nq)
        D, I = _search(idx, X, Q, k, what, expect, reconstruct=nq <= 7, ids=finite)
        assert np.isin(I, finite).all(), what
        assert I[0, 0] == 1 and I[1, 0] == 4 and I[2, 0] == N - 2, what
        if nq > 3:
            assert np.array_equal(I[3], finite[:k]), what + ": zero query"
        if expect[0] == HI_ONLY:
            assert idx.last_hi_only_fallbacks() == nq, what


@pytest.mark.timeout(300)
def test_nan_rows_padding():
    """Fewer finite rows than k: the finite rows, then -1 / -FLT_MAX, on every path (4096 rows, 30 of them finite,
    for the tensor scans; 50 rows, 5 finite, for the FMA scans)."""
    d, k = 520, 40
    for n, keep, paths in ((50, [2, 17, 31, 32, 49], _nan_paths(d)[:4]), (4096, list(range(4066, 4096)), _nan_paths(d)[4:])):
        X, finite = _with_nan_rows(_rows(n, d), [i for i in range(n) if i not in keep], {})
        assert np.array_equal(finite, keep)
        idx = _index(d, X=X)
        for flags, nq, expect in paths:
            Q = _queries(nq, d)
            idx.set_tensor_scan(flags)
            D, I = _search(idx, X, Q, k, "n %d flags %d nq %d" % (n, flags, nq), expect, reconstruct=nq <= 7, ids=finite)
            assert (I[:, :len(keep)] >= 0).all() and (I[:, len(keep):] == -1).all()
            assert (D[:, len(keep):] == knn_ref.NEG).all()


# ---- range search -----------------------------------------------------------------------------------------------

@pytest.mark.timeout(300)
@pytest.mark.parametrize("d", RANGE_WIDTHS)
def test_range_every_width(d):
    """range_scan_kernel<CH> for CH = 1..8 with partial chunks: no hits, a few, and more than the first capacity of
    4096 (the regrow path), ids equal to float64 except within TOL of the threshold; NaN rows never returned.  A
    basis-vector query makes every score exact: the hits must be exactly the rows whose coordinate is > thresh, so
    a row equal to the threshold is excluded (FAISS's strict >) and the next fp16 value above it is included."""
    n = 20011
    X, finite = _with_nan_rows(_rows(n, d), [7, n - 1], {100: d - 1, 101: 0})
    j, thr = d - 1, 0.25
    at, above = 2000, 2001
    X[at, j] = np.float16(thr)
    X[above, j] = np.nextafter(np.float16(thr), np.float16(1))
    idx = _index(d, X=X)
    Q = _queries(3, d)
    S64 = knn_ref.scores_f64(X, Q)
    s0 = np.sort(S64[0, finite])[::-1]
    for t in (1.5, float(s0[9] + s0[10]) / 2, 0.0):
        lims, D, I = idx.range_search(Q, t)
        assert lims.dtype == np.uint64 and lims.shape == (4,)
        for q in range(3):
            ids = I[lims[q]:lims[q + 1]]
            assert np.all(np.diff(ids) > 0), "d %d thr %g query %d: ids not ascending" % (d, t, q)
            assert np.isin(ids, finite).all(), "d %d: a NaN row was returned" % d
            want = set(finite[S64[q, finite] > t].tolist())
            for i in set(ids.tolist()) ^ want:
                assert abs(S64[q, i] - t) <= TOL, "d %d thr %g query %d: id %d differs, not at the threshold" % (d, t, q, i)
            np.testing.assert_allclose(D[lims[q]:lims[q + 1]], S64[q, ids], atol=TOL)
        if t == 1.5:
            assert lims[-1] == 0
        elif t == 0.0:
            assert min(np.diff(lims.astype(np.int64))) > 4096
        else:
            assert 5 <= lims[1] <= 15
    e = np.zeros((1, d), np.float32)
    e[0, j] = 1.0
    lims, D, I = idx.range_search(e, thr)
    col = X[finite, j].astype(np.float32)
    want = finite[col > np.float32(thr)]
    assert np.array_equal(I, want), "d %d: basis query: %d hits, expected %d (row at the threshold returned: %s)" % (
        d, I.size, want.size, at in I)
    assert above in I and at not in I
    assert np.array_equal(D, X[want, j].astype(np.float32))


# ---- shard merge at its limits ----------------------------------------------------------------------------------

@pytest.mark.timeout(300)
def test_merge_at_its_limits():
    """merge_shard_results at G * k = 16384 (G = 2, k = 8192) against the oracle merge, bit for bit, with shards
    holding fewer than k results and equal scores in different shards (ascending global id wins); G * k = 16385 is
    refused."""
    import torch
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(5)
    G, nq, k = 2, 3, 8192
    Dg = -np.sort(-rng.standard_normal((G, nq, k)).astype(np.float32), axis=2)
    Ig = np.stack([rng.permutation(10 * k)[:k] + g * 10 * k for g in range(G)]).reshape(G, 1, k).repeat(nq, axis=1)
    Ig = Ig.astype(np.int64)
    # query 0: every score of shard 0 also in shard 1, shard 1 holding the lower id of each pair
    Dg[1, 0] = Dg[0, 0]
    Ig[1, 0] = 2 * Ig[0, 0]
    Ig[0, 0] = 2 * Ig[0, 0] + 1
    # query 1: shard 1 holds 100 results, shard 0 holds 3000; query 2: shard 0 holds none
    Dg[1, 1, 100:], Ig[1, 1, 100:] = knn_ref.NEG, -1
    Dg[0, 1, 3000:], Ig[0, 1, 3000:] = knn_ref.NEG, -1
    Dg[0, 2], Ig[0, 2] = knn_ref.NEG, -1
    D, I = m.merge_shard_results(torch.from_numpy(Dg).cuda(), torch.from_numpy(Ig).cuda(), k)
    D, I = D.cpu().numpy(), I.cpu().numpy()
    Do, Io = knn_ref.merge_shards(Dg, Ig, k)
    assert np.array_equal(I, Io) and np.array_equal(D, Do)
    assert np.array_equal(I[0, 0:2], sorted(Ig[:, 0, 0])) and D[0, 0] == D[0, 1]
    assert (I[1, :3100] >= 0).all() and (I[1, 3100:] == -1).all() and (D[1, 3100:] == knn_ref.NEG).all()
    G, k = 5, 3277   # 16385 candidates per query
    with pytest.raises(m.B200Error, match="exceeds 16384"):
        m.merge_shard_results(torch.zeros((G, 1, k), device="cuda"), torch.zeros((G, 1, k), dtype=torch.int64, device="cuda"), k)
