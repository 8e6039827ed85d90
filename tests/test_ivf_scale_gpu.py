"""IVF-Flat at serving shapes against a float64 ranking of the probed lists (oracle/knn_ref.ivf_check).

What tests/test_ivf_gpu.py does not reach: the wgmma coarse scan (nlist >= 4096) in split and hi-only mode,
the 256-query batches of the list scan, every row width (CH = 1..8, partial 256-column chunks) of the
assignment, list-scan and range kernels, segmented / skewed / empty / short lists, k up to the 8192 maximum,
and ties between identical rows held in different lists (equal scores come back by ascending id).

A query whose nprobe-th and (nprobe+1)-th float64 centroid scores are closer than 1e-5 may have been given
either list by the coarse scan: it is skipped if it does not match the float64 probes, and is left out of the
FMA-vs-wgmma and batch-vs-single comparisons.  At most 5 % of the queries of a test may be skipped.  Rows are regenerated on
the host (oracle/synth_ref), never read back through the index under test.
"""
import numpy as np
import pytest

from oracle import knn_ref, synth_ref

pytestmark = pytest.mark.gpu
TOL = 2e-6
CHUNK = 16384


def _rows(n, d, **spec):
    """Synthetic rows 0..n-1 regenerated on the host in chunks (bounded temporaries)."""
    return np.concatenate([synth_ref.rows_f16(min(CHUNK, n - s), d, row0=s, **spec) for s in range(0, n, CHUNK)])


def _graph_search(idx, Q, k, reconstruct=False):
    """nq <= 4 queries through search_device: the first call of a shape runs eagerly, the second replays the
    CUDA graph captured for it."""
    import torch

    t = torch.from_numpy(np.ascontiguousarray(Q, dtype=np.float32).reshape(-1, idx.d)).cuda()
    idx.search_device(t, k, reconstruct=reconstruct)
    out = idx.search_device(t, k, reconstruct=reconstruct)
    return [o.cpu().numpy() for o in out]


def _assign_of(idx, n):
    """The list of every row id, as the index holds it."""
    sizes, ids = idx.invlists()
    got = np.full(n, -1, dtype=np.int64)
    got[ids - idx.id_base] = np.repeat(np.arange(idx.nlist), sizes)
    return got


class _Skips:
    def __init__(self):
        self.asked = self.checked = 0

    def add(self, nq, checked):
        self.asked += nq
        self.checked += checked

    def assert_few(self):
        assert self.asked - self.checked <= 0.05 * self.asked, "%d of %d queries skipped" % (
            self.asked - self.checked, self.asked)


def _check(D, I, X, assign, C16, Q, k, nprobe, skips, what, id_base=0):
    ok, msg, checked = knn_ref.ivf_check(D, I, X, assign, C16, Q, k, nprobe, tol=TOL, id_base=id_base)
    assert ok, "%s: %s" % (what, msg)
    skips.add(Q.shape[0], checked)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("nlist,d,nqs", [
    (4095, 768, (5, 64, 128, 129, 300, 1000)),   # FMA coarse scan
    (4096, 768, (5, 64, 128, 129, 300, 1000)),   # wgmma coarse scan: split mode, hi-only above 128 queries
    (4096, 1024, (64,)),                         # the e2e shape (ViT-H/14)
], ids=["nlist4095-d768", "nlist4096-d768", "nlist4096-d1024"])
def test_ivf_coarse_paths(nlist, d, nqs):
    """The coarse step at benchmark size: the wgmma centroid scan (nlist >= 4096, nq > 4, nprobe <= 128) in
    split mode and, above 128 queries with nprobe <= 64, the hi-only pass with its exact re-score and proof;
    nprobe 129 goes back to the FMA scan.  Each search also runs with the FMA scan forced, which must give
    the same ids, and single queries (the CUDA-graph path) must reproduce their rows of the batch."""
    import clip_retrieval_b200 as m

    n, cs = 32 * nlist, 9
    kw = dict(seed=21, clustered=True, centroid_seed=cs, nlist=nlist)
    C32 = synth_ref.centroids_f32(nlist, d, cs)
    C16 = C32.astype(np.float16)
    idx = m.B200IVFFlatIndex(d, nlist, C32)
    idx.add_synthetic(n, m.SynthSpec(cw=3, nw=1, **kw))
    X = _rows(n, d, **kw)
    assign = synth_ref.list_of_rows(cs, np.arange(n), nlist)
    assert np.array_equal(idx.invlists()[0], np.bincount(assign, minlength=nlist))
    Q = synth_ref.rows_f32(max(nqs), d, seed=31, clustered=True, centroid_seed=cs, nlist=nlist)
    skips = _Skips()
    for i, nprobe in enumerate((16, 64, 100, 129)):
        idx.nprobe = nprobe
        for j, nq in enumerate(nqs):
            if nq == 1000 and nprobe > 64:
                continue   # 300 queries already cover these paths; 1000 is for the hi-only pass
            k = (1, 40, 128)[(i + j) % 3]
            what = "nprobe %d nq %d k %d" % (nprobe, nq, k)
            q = Q[:nq]
            idx.set_tensor_scan(True)
            D, I = idx.search(q, k)
            if nq > 128 and nprobe <= 64:
                assert idx.last_hi_only_fallbacks() == 0, what   # iid centroids: the hi-only proof holds
            _check(D, I, X, assign, C16, q, k, nprobe, skips, what)
            keep = knn_ref.probes_f64(C16, q, nprobe)[1]
            idx.set_tensor_scan(False)
            Df, If = idx.search(q, k)
            assert np.array_equal(If[keep], I[keep]), what
            np.testing.assert_allclose(Df[keep], D[keep], atol=TOL, err_msg=what)
            idx.set_tensor_scan(True)
            if nq == 1000:
                for r in (0, 1, nq - 1):
                    if keep[r]:
                        Ds, Is = _graph_search(idx, q[r], k)
                        assert np.array_equal(Is[0], I[r]) and np.array_equal(Ds[0], D[r]), (what, r)
    skips.assert_few()


@pytest.mark.timeout(300)
def test_ivf_list_scan_query_batches():
    """The list scan runs 256 queries per launch, offsetting queries, probes and output keys by the batch start:
    nq on both sides of 256 and 512, checked query by query, and rows at the batch seams against single queries."""
    import clip_retrieval_b200 as m

    d, nlist, n, k, nprobe, cs = 256, 37, 30000, 40, 4, 5
    kw = dict(seed=41, clustered=True, centroid_seed=cs, nlist=nlist)
    C32 = synth_ref.centroids_f32(nlist, d, cs)
    C16 = C32.astype(np.float16)
    idx = m.B200IVFFlatIndex(d, nlist, C32)
    idx.add_synthetic(n, m.SynthSpec(cw=3, nw=1, **kw))
    X = _rows(n, d, **kw)
    assign = synth_ref.list_of_rows(cs, np.arange(n), nlist)
    Q = synth_ref.rows_f32(513, d, seed=43, clustered=True, centroid_seed=cs, nlist=nlist)
    idx.nprobe = nprobe
    skips = _Skips()
    for nq in (255, 256, 257, 513):
        D, I = idx.search(Q[:nq], k)
        _check(D, I, X, assign, C16, Q[:nq], k, nprobe, skips, "nq %d" % nq)
    keep = knn_ref.probes_f64(C16, Q, nprobe)[1]
    for r in (255, 256, 512):
        if keep[r]:
            Ds, Is = _graph_search(idx, Q[r], k)
            assert np.array_equal(Is[0], I[r]) and np.array_equal(Ds[0], D[r]), r
    skips.assert_few()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("d", [64, 200, 264, 520, 1024, 1280, 1536, 1792, 2048])
def test_ivf_every_row_width(d):
    """CH = ceil(d / 256) = 1..8, with partial chunks (d = 200, 264, 520): the argmax assignment of `add` over
    nlist = 37 (not a multiple of 4), search at nprobe 1 and 4, and range_search."""
    import clip_retrieval_b200 as m

    nlist, n, k, cs = 37, 4000, 40, 3
    kw = dict(seed=51, clustered=True, centroid_seed=cs, nlist=nlist)
    X = synth_ref.rows_f16(n, d, **kw)
    C32 = synth_ref.centroids_f32(nlist, d, cs)
    C16 = C32.astype(np.float16)
    idx = m.B200IVFFlatIndex(d, nlist, C32)
    idx.add(X)
    got = _assign_of(idx, n)
    ref = knn_ref.ivf_assign(X, C16)
    Sx = np.sort(knn_ref.scores_f64(C16, X.astype(np.float32)), axis=1)
    bad = np.nonzero(got != ref)[0]
    assert np.all(Sx[bad, -1] - Sx[bad, -2] < 1e-5), "rows %s are in another list than the argmax" % bad[:8]
    assert (np.bincount(got, minlength=nlist) > 0).all()   # the last lists of the 4-list groups are filled too
    Q = synth_ref.rows_f32(8, d, seed=53, clustered=True, centroid_seed=cs, nlist=nlist)
    skips = _Skips()
    for nprobe in (1, 4):
        idx.nprobe = nprobe
        D, I, R = idx.search_and_reconstruct(Q, k)
        _check(D, I, X, got, C16, Q, k, nprobe, skips, "d %d nprobe %d" % (d, nprobe))
        assert np.array_equal(R[I >= 0], X[I[I >= 0]].astype(np.float32))
    thr = 0.85
    lims, Dr, Ir = idx.range_search(Q, thr)
    _check_range(lims, Dr, Ir, X, got, C16, Q, 4, thr)
    assert lims[-1] > 0
    skips.assert_few()


def _check_range(lims, D, I, X, assign, C16, Q, nprobe, thr, id_base=0):
    """Hits = rows of the float64 probes scoring above thr, ids ascending; a row within TOL of thr may go either way."""
    probes, keep = knn_ref.probes_f64(C16, Q, nprobe)
    for q in np.nonzero(keep)[0]:
        rows = np.nonzero(np.isin(assign, probes[q]))[0]
        s = knn_ref.scores_f64(X[rows], Q[q:q + 1])[0]
        want = set((rows[s > thr] + id_base).tolist())
        got = I[lims[q]:lims[q + 1]]
        assert np.all(np.diff(got) > 0), q
        S = dict(zip((rows + id_base).tolist(), s))
        for i in set(got.tolist()) ^ want:
            assert i in S and abs(S[i] - thr) <= TOL, "query %d: id %d differs and is not at the threshold" % (q, i)
        np.testing.assert_allclose(D[lims[q]:lims[q + 1]], [S[i] for i in got.tolist()], atol=TOL)


@pytest.mark.timeout(300)
def test_ivf_skewed_empty_and_short_lists():
    """Explicit lists (an index file's own): one list holds 60 % of the rows, so one query splits it into 32
    segments while short lists get segments that start past their end; lists of 1, 2, 3, 5 and 7 rows; a
    quarter of the lists empty, with queries that probe them; k beyond the rows held (-1 padding)."""
    import clip_retrieval_b200 as m

    d, nlist, n = 128, 64, 60000
    X = synth_ref.rows_f16(n, d, seed=61)
    C32 = synth_ref.centroids_f32(nlist, d, 13)
    C16 = C32.astype(np.float16)
    rng = np.random.default_rng(0)
    sizes = np.zeros(nlist, dtype=np.int64)
    sizes[0] = 36001                                  # 60 %, not a multiple of 4
    sizes[1:6] = (1, 2, 3, 5, 7)
    rest = n - sizes.sum()                            # lists 6..47 share the rest; 48..63 stay empty
    cut = np.sort(rng.choice(np.arange(1, rest), 41, replace=False))
    sizes[6:48] = np.diff(np.concatenate([[0], cut, [rest]]))
    assert sizes.sum() == n and (sizes[48:] == 0).all()
    assign = np.repeat(np.arange(nlist), sizes)[rng.permutation(n)]
    idx = m.B200IVFFlatIndex(d, nlist, C32)
    idx.add_with_lists(X, assign)
    assert np.array_equal(idx.invlists()[0], sizes)
    # queries next to chosen centroids: the long list, empty lists, the short lists, ordinary lists
    targets = np.array([0, 50, 1, 2, 3, 4, 5, 63, 6, 48, 20, 0, 55, 5, 1, 30, 47])
    noise = synth_ref.rows_f32(17, d, seed=63)
    Q = C32[targets] + 0.3 * noise
    Q = (Q / np.linalg.norm(Q, axis=1, keepdims=True)).astype(np.float32)
    skips = _Skips()
    for nprobe in (1, 4, 16):
        idx.nprobe = nprobe
        for nq in (1, 3, 17):
            for k in (40, 1000):
                D, I = idx.search(Q[:nq], k)
                _check(D, I, X, assign, C16, Q[:nq], k, nprobe, skips, "nprobe %d nq %d k %d" % (nprobe, nq, k))
                if nprobe == 1:   # probe = the target list: -1 padding past what it holds
                    for q in range(nq):
                        held = sizes[targets[q]]
                        assert (I[q, :min(k, held)] >= 0).all() and (I[q, held:] == -1).all(), (q, held)
    # range_search over the long list (more hits than the first capacity of 4096)
    idx.nprobe = 1
    lims, Dr, Ir = idx.range_search(Q[:1], 0.0)
    assert lims[-1] > 4096
    _check_range(lims, Dr, Ir, X, assign, C16, Q[:1], 1, 0.0)
    skips.assert_few()


@pytest.mark.timeout(600)
def test_ivf_large_k():
    """k from 129 to the 8192 maximum: the list-scan block shrinks to 128 threads above k = 2560 and to 64
    above 5120, and the level-2 select runs over several chunks; 8193 is refused."""
    import clip_retrieval_b200 as m

    d, nlist, n, nprobe, cs = 128, 37, 40000, 12, 11
    kw = dict(seed=71, clustered=True, centroid_seed=cs, nlist=nlist)
    C32 = synth_ref.centroids_f32(nlist, d, cs)
    C16 = C32.astype(np.float16)
    idx = m.B200IVFFlatIndex(d, nlist, C32)
    idx.add_synthetic(n, m.SynthSpec(cw=3, nw=1, **kw))
    X = _rows(n, d, **kw)
    assign = synth_ref.list_of_rows(cs, np.arange(n), nlist)
    sizes = np.bincount(assign, minlength=nlist)
    Q = synth_ref.rows_f32(300, d, seed=73, clustered=True, centroid_seed=cs, nlist=nlist)
    idx.nprobe = nprobe
    probes = knn_ref.probes_f64(C16, Q, nprobe)[0]
    assert sizes[probes].sum(axis=1).min() >= 8192   # every k is filled
    skips = _Skips()
    for nq in (1, 9, 300):
        for k in (129, 1000, 2561, 5121, 8192):
            D, I = idx.search(Q[:nq], k)
            sel = np.arange(nq) if nq < 300 or k <= 1000 else np.r_[0:nq:10, nq - 1]   # bound the host check
            _check(D[sel], I[sel], X, assign, C16, Q[sel], k, nprobe, skips, "nq %d k %d" % (nq, k))
    with pytest.raises(ValueError):
        idx.search(Q[:1], 8193)
    skips.assert_few()


@pytest.mark.timeout(300)
def test_ivf_ties_by_ascending_id():
    """Identical rows held in different lists, in the reverse of their id order (explicit lists, then a second
    batch with one explicit list and one argmax row): equal scores must come back by ascending id, through
    the CUDA-graph path (nq <= 4) and a batch of 300, with id_base = 10**10; reconstruction stays exact."""
    import clip_retrieval_b200 as m

    d, nlist, n, cs, base = 128, 8, 3000, 17, 10**10
    kw = dict(seed=81, clustered=True, centroid_seed=cs, nlist=nlist)
    C32 = synth_ref.centroids_f32(nlist, d, cs)
    C16 = C32.astype(np.float16)
    X = np.concatenate([synth_ref.rows_f16(n, d, **kw), synth_ref.rows_f16(500, d, row0=n, **kw)])
    copies = np.array([10, 500, 1500, 2999, n + 100, n + 400])
    X[copies] = X[10]
    lists = knn_ref.ivf_assign(X, C16)
    lists[copies[:5]] = (7, 5, 3, 1, 0)     # the lowest id sits in the last list, the highest explicit one first
    idx = m.B200IVFFlatIndex(d, nlist, C32)
    idx.add_with_lists(X[:n], lists[:n])
    idx.finalize()
    idx.add_with_lists(X[n:n + 300], lists[n:n + 300])
    idx.add(X[n + 300:])                    # bucketed by argmax, copy n + 400 among them
    idx.finalize()
    idx.id_base = base
    got = _assign_of(idx, X.shape[0])
    assert np.array_equal(got[:n + 300], lists[:n + 300])
    assert len(set(got[copies].tolist())) >= 5
    idx.nprobe = nlist
    r = X[10].astype(np.float32)
    want = copies + base                    # ascending
    for k in (1, 10):
        for nq in (1, 4):
            D, I, R = idx.search_and_reconstruct(np.tile(r, (nq, 1)), k)
            assert (I[:, :min(k, 6)] == want[:min(k, 6)]).all(), (k, nq, I[:, :6])
            assert (D[:, :min(k, 6)] == D[0, 0]).all()
            assert np.array_equal(R, X[I - base].astype(np.float32))
            Ds, Is, Rs = _graph_search(idx, np.tile(r, (nq, 1)), k, reconstruct=True)
            assert np.array_equal(Is, I) and np.array_equal(Ds, D) and np.array_equal(Rs, R)
    Q = synth_ref.rows_f32(300, d, seed=83, clustered=True, centroid_seed=cs, nlist=nlist)
    Q[[0, 150, 299]] = r
    skips = _Skips()
    for k in (1, 10):
        D, I, R = idx.search_and_reconstruct(Q, k)
        assert (I[[0, 150, 299], :min(k, 6)] == want[:min(k, 6)]).all(), k
        _check(D, I, X, got, C16, Q, k, nlist, skips, "nq 300 k %d" % k, id_base=base)
        assert np.array_equal(R, X[I - base].astype(np.float32))
    for i in np.concatenate([copies, [0, n - 1, n + 499]]):
        assert np.array_equal(idx.reconstruct(base + int(i)), X[i].astype(np.float32))
    skips.assert_few()
