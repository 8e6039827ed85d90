"""Parity of the CUDA search path (through the C ABI) against the CPU oracle.

Integer/index work is bit-exact where the arithmetic allows it (synthetic rows, ids under exact
ties, reconstructed rows); scores are fp32 sums over d terms evaluated in a different order than
the oracle's, so ids are compared tie-aware: identical except where the float64 scores of the
swapped ids differ by <= TOL (oracle/knn_ref.check_topk).
"""
import numpy as np
import pytest

from oracle import knn_ref, synth_ref

pytestmark = pytest.mark.gpu
TOL = 2e-6  # |fp32 sum - exact| for unit vectors, d <= 1024 (observed ~2e-7)


@pytest.fixture(scope="module")
def b200():
    import clip_retrieval_b200 as m

    return m


def _queries(nq, d, seed=4321):
    return synth_ref.rows_f32(nq, d, seed=seed)


def test_synthetic_rows_bit_exact(b200):
    from clip_retrieval_b200.index import synth_rows

    for d in (64, 768):
        for spec, kw in (
            (b200.SynthSpec(seed=1234), dict(seed=1234)),
            (b200.SynthSpec(seed=99, clustered=True, centroid_seed=7, nlist=37, cw=3, nw=1),
             dict(seed=99, clustered=True, centroid_seed=7, nlist=37, cw=3, nw=1)),
        ):
            got16 = synth_rows(513, d, spec, row0=1000, dtype="float16").cpu().numpy()
            got32 = synth_rows(513, d, spec, row0=1000, dtype="float32").cpu().numpy()
            assert np.array_equal(got16.view(np.uint16), synth_ref.rows_f16(513, d, 1000, **kw).view(np.uint16))
            assert np.array_equal(got32.view(np.uint32), synth_ref.rows_f32(513, d, 1000, **kw).view(np.uint32))


@pytest.mark.parametrize("d", [64, 512, 768, 1024])
@pytest.mark.parametrize("nq", [1, 2, 3, 5, 9])
def test_flat_search_matches_oracle(b200, d, nq):
    n, k = 20011, 40
    X = synth_ref.rows_f16(n, d)
    Q = _queries(nq, d)
    idx = b200.B200FlatIndex(d)
    idx.add(X)
    assert idx.ntotal == n and idx.d == d
    D, I = idx.search(Q, k)
    assert D.dtype == np.float32 and I.dtype == np.int64 and D.shape == (nq, k)
    ok, msg, strict = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg
    assert strict == nq, "ids differ from the float64 ranking in %d queries (near-ties)" % (nq - strict)
    Do, Io = knn_ref.flat_search(X, Q, k)
    np.testing.assert_allclose(D, Do, rtol=0, atol=TOL)


def test_search_and_reconstruct_and_padding(b200):
    d, n, k = 768, 25, 40  # k > ntotal: -1 padding the reference truncates at (clip_back.py:370-375)
    X = synth_ref.rows_f16(n, d)
    Q = _queries(3, d)
    idx = b200.B200FlatIndex(d)
    idx.add(X[:10])
    idx.add(X[10:].astype(np.float32))  # fp32 add path rounds to the same fp16
    D, I, R = idx.search_and_reconstruct(Q, k)
    ok, msg, _ = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg
    assert np.all(I[:, n:] == -1) and np.all(D[:, n:] == knn_ref.NEG)
    Ro = knn_ref.reconstruct(X, I)
    assert np.array_equal(R[:, :n], Ro[:, :n])      # stored rows upcast: bit exact
    assert np.all(np.isnan(R[:, n:]))


def test_empty_index_and_empty_query(b200):
    idx = b200.B200FlatIndex(64)
    D, I = idx.search(_queries(2, 64), 5)
    assert np.all(I == -1) and np.all(D == knn_ref.NEG)
    idx.add(synth_ref.rows_f16(100, 64))
    D, I = idx.search(np.zeros((0, 64), np.float32), 5)
    assert D.shape == (0, 5) and I.shape == (0, 5)
    with pytest.raises(AssertionError):
        idx.search(np.zeros((1, 32), np.float32), 5)


def test_exact_ties_break_by_lower_id(b200):
    d, k = 128, 10
    base = synth_ref.rows_f16(50, d)
    X = np.concatenate([base, base, base[:7]])  # every row duplicated (some three times)
    Q = base[:4].astype(np.float32)
    idx = b200.B200FlatIndex(d)
    idx.add(X)
    D, I = idx.search(Q, k)
    Do, Io = knn_ref.flat_search(X, Q, k)
    ok, msg, _ = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg
    for q in range(4):  # the duplicates of the query row itself are exact ties at the top
        assert I[q, 0] == q and I[q, 1] == q + 50
        assert D[q, 0] == D[q, 1]


@pytest.mark.parametrize("k", [1, 7, 100, 1000, 3000])
def test_k_range(b200, k):
    d, n = 256, 30000
    X = synth_ref.rows_f16(n, d)
    Q = _queries(2, d)
    idx = b200.B200FlatIndex(d)
    idx.add(X)
    D, I = idx.search(Q, k)
    ok, msg, _ = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg


def test_id_base_and_device_buffers(b200):
    import torch

    d, n, k = 768, 5000, 40
    X = synth_ref.rows_f16(n, d)
    Q = _queries(4, d)
    idx = b200.B200FlatIndex(d)
    idx.add(torch.from_numpy(X).cuda())
    idx.id_base = 10_000_000_000
    D, I, R = idx.search_device(torch.from_numpy(Q).cuda(), k, reconstruct=True)
    D, I, R = D.cpu().numpy(), I.cpu().numpy(), R.cpu().numpy()
    ok, msg, _ = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, id_base=10_000_000_000, tol=TOL)
    assert ok, msg
    assert np.array_equal(R, knn_ref.reconstruct(X, I, id_base=10_000_000_000))
    ms, launches = idx.last_scan_ms()
    assert launches >= 1 and ms > 0


def test_library_generated_index_equals_host_rows(b200):
    d, n, k = 768, 40000, 40
    spec = b200.SynthSpec(seed=1234)
    idx = b200.B200FlatIndex(d)
    idx.reserve(n)
    idx.add_synthetic(n // 2, spec, row0=0)
    idx.add_synthetic(n - n // 2, spec, row0=n // 2)
    X = synth_ref.rows_f16(n, d)
    Q = _queries(6, d)
    D, I, R = idx.search_and_reconstruct(Q, k)
    ok, msg, _ = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg
    assert np.array_equal(R, knn_ref.reconstruct(X, I))


def test_merge_of_shard_candidates(b200):
    import torch

    d, n, k, G = 256, 12000, 40, 4
    X = synth_ref.rows_f16(n, d)
    Q = _queries(5, d)
    per = n // G
    Dg, Ig = [], []
    for g in range(G):
        idx = b200.B200FlatIndex(d)
        idx.add(X[g * per:(g + 1) * per])
        idx.id_base = g * per
        Dd, Id = idx.search_device(torch.from_numpy(Q).cuda(), k)
        Dg.append(Dd)
        Ig.append(Id)
    Dg, Ig = torch.stack(Dg), torch.stack(Ig)
    D, I = b200.merge_shard_results(Dg, Ig, k)
    Do, Io = knn_ref.merge_shards(Dg.cpu().numpy(), Ig.cpu().numpy(), k)
    assert np.array_equal(I.cpu().numpy(), Io) and np.array_equal(D.cpu().numpy(), Do)  # pure selection: exact
    ok, msg, _ = knn_ref.check_topk(D.cpu().numpy(), I.cpu().numpy(), knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg


def test_full_size_properties_sharded_idempotent(b200):
    """Size-independent property at a size the oracle cannot rank: the top-k of the whole equals
    the merge of the top-k of its halves, and searching twice is idempotent."""
    import torch

    d, n, k = 768, 3_000_000, 40
    spec = b200.SynthSpec(seed=5)
    whole = b200.B200FlatIndex(d)
    whole.add_synthetic(n, spec)
    Q = torch.from_numpy(_queries(8, d)).cuda()
    D1, I1 = whole.search_device(Q, k)
    D2, I2 = whole.search_device(Q, k)
    assert torch.equal(I1, I2) and torch.equal(D1, D2)
    halves = []
    for g in range(2):
        h = b200.B200FlatIndex(d)
        h.add_synthetic(n // 2, spec, row0=g * (n // 2))
        h.id_base = g * (n // 2)
        halves.append(h.search_device(Q, k))
    Dm, Im = b200.merge_shard_results(torch.stack([h[0] for h in halves]), torch.stack([h[1] for h in halves]), k)
    assert torch.equal(Im, I1) and torch.equal(Dm, D1)
    # spot-check the winners against exact scores of the regenerated rows
    ids = I1.cpu().numpy()
    for q in range(2):
        rows = np.stack([synth_ref.rows_f16(1, d, int(i), seed=5)[0] for i in ids[q, :5]])
        s = rows.astype(np.float64) @ Q[q].cpu().numpy().astype(np.float64)
        np.testing.assert_allclose(D1[q, :5].cpu().numpy(), s, atol=TOL)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("nq,k,n,d", [(5, 40, 4096, 768), (64, 40, 60000, 768), (130, 128, 50021, 768), (300, 1, 33000, 512),
                                      (1000, 40, 150000, 768), (17, 40, 20000, 1024),
                                      (40, 40, 30011, 200), (300, 40, 30011, 1280), (64, 64, 20000, 2048)])
def test_tensor_scan_matches_oracle_and_fma_scan(b200, nq, k, n, d):
    """The wgmma batch scan (fp32 query split into fp16 hi/lo) against the float64 ranking and
    against the FMA scan of the same index.  d = 200 ends inside a 64-column TMA box (zero-filled K tail);
    d = 1280 and 2048 run past 1024 columns."""
    X = synth_ref.rows_f16(n, d)
    Q = _queries(nq, d)
    idx = b200.B200FlatIndex(d)
    idx.add(X)
    D, I = idx.search(Q, k)                 # nq > 4, k <= 128 -> tensor path
    ok, msg, strict = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg
    idx.set_tensor_scan(False)
    Df, If = idx.search(Q, k)
    ok, msg, _ = knn_ref.check_topk(Df, If, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg
    np.testing.assert_allclose(D, Df, atol=TOL)
    assert (I == If).mean() > 0.995         # ids agree except across near-ties


@pytest.mark.timeout(300)
@pytest.mark.parametrize("nq,k,n,d", [(129, 40, 50021, 768), (300, 40, 200000, 768), (1000, 10, 150000, 512),
                                      (257, 64, 33000, 1024), (200, 40, 30011, 200), (257, 40, 30011, 1280),
                                      (300, 10, 20000, 2048)])
def test_hi_only_scan_is_exact(b200, nq, k, n, d):
    """More than 128 queries: approximate hi-only wgmma pass + exact re-score + per-query proof
    (knn_mma.cu).  Must equal the float64 ranking and the split-mode scan of the same index."""
    X = synth_ref.rows_f16(n, d)
    Q = _queries(nq, d)
    idx = b200.B200FlatIndex(d)
    idx.add(X)
    S64 = knn_ref.scores_f64(X, Q)
    D, I = idx.search(Q, k)
    ok, msg, _ = knn_ref.check_topk(D, I, S64, k, tol=TOL)
    assert ok, msg
    assert idx.last_hi_only_fallbacks() == 0            # iid rows: every proof succeeds
    idx.set_tensor_scan(1 | 8)                          # split mode only
    Ds, Is = idx.search(Q, k)
    ok, msg, _ = knn_ref.check_topk(Ds, Is, S64, k, tol=TOL)
    assert ok, msg
    np.testing.assert_allclose(D, Ds, atol=TOL)
    assert (I == Is).mean() > 0.995


@pytest.mark.timeout(300)
def test_hi_only_scan_falls_back_on_packed_duplicates(b200):
    """Rows that are exact copies of each other tie inside the error bound of the approximate pass:
    the proof must fail for the queries whose k-th neighbour sits in such a pack, those queries are
    re-run in split mode, and the result (ties by ascending id) is still exact."""
    d, k, nq = 768, 40, 200
    base = synth_ref.rows_f16(5000, d)
    X = np.concatenate([base, np.repeat(base[:40], 100, axis=0), base[::-1]])   # 100 copies of 40 rows + a mirrored copy
    Q = _queries(nq, d)
    Q[:8] = 0.25 * base[:8].astype(np.float32) + 1e-3 * Q[:8]   # queries that land on the packed rows
    idx = b200.B200FlatIndex(d)
    idx.add(X)
    D, I = idx.search(Q, k)
    ok, msg, _ = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg
    assert idx.last_hi_only_fallbacks() >= 8
    idx.set_tensor_scan(False)
    Df, If = idx.search(Q, k)
    assert np.array_equal(I[:8], If[:8])                # exact ties: ascending ids in both paths
    np.testing.assert_allclose(D, Df, atol=TOL)


def test_range_search_matches_oracle(b200):
    """index.range_search (clip_filter.py:52): ids identical to the oracle except for rows whose exact
    score lies within TOL of the threshold."""
    d, n = 768, 30000
    X = synth_ref.rows_f16(n, d)
    Q = _queries(3, d)
    idx = b200.B200FlatIndex(d)
    idx.add(X)
    S64 = knn_ref.scores_f64(X, Q)
    for thr in (0.08, 0.02, 0.5):   # few hits, thousands of hits (buffer regrowth), none
        lims, D, I = idx.range_search(Q, thr)
        lo, Do, Io = knn_ref.range_search(X, Q, thr)
        assert lims.dtype == np.uint64 and lims.shape == (4,)
        for q in range(3):
            got = set(I[lims[q]:lims[q + 1]].tolist())
            ref = set(Io[lo[q]:lo[q + 1]].tolist())
            for i in got ^ ref:
                assert abs(S64[q, i] - thr) <= TOL, "id %d differs and is not at the threshold" % i
            ids = I[lims[q]:lims[q + 1]]
            assert np.all(np.diff(ids) > 0)
            np.testing.assert_allclose(D[lims[q]:lims[q + 1]], S64[q, ids], atol=TOL)


def test_load_index_on_writer_format_shards(b200, tmp_path):
    """a10: `load_index(folder)` (clip_back.py:589-596 counterpart) on fp16 shards named as the reference writer
    names them (`img_emb_{id:0{w}d}.npy`, writer.py:22,67-87); rows land in sorted-file order = global id order."""
    d, k = 512, 10
    X = synth_ref.rows_f16(3000, d)
    parts = [X[:1000], X[1000:1100], X[1100:]]
    folder = tmp_path / "img_emb"
    folder.mkdir()
    for i, p in enumerate(parts):
        np.save(str(folder / ("img_emb_%02d.npy" % i)), p)
    (folder / "ignored.txt").write_text("x")
    idx = b200.load_index(str(folder), enable_faiss_memory_mapping=True)
    assert idx.ntotal == 3000 and idx.d == d
    Q = _queries(4, d)
    D, I, R = idx.search_and_reconstruct(Q, k)
    ok, msg, strict = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok and strict == 4, msg
    assert np.array_equal(R, knn_ref.reconstruct(X, I))
    one = b200.load_index(str(folder / "img_emb_01.npy"))
    assert one.ntotal == 100
    with pytest.raises(ValueError):
        b200.load_index(str(tmp_path))                    # no shard there
    with pytest.raises(ValueError):
        idx.search(Q, 9000)                               # k above the supported maximum: a clear error, not a CUDA one
