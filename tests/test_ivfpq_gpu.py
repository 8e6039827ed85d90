"""IVF-PQ search on the GPU (csrc/knn_ivfpq.cu) against the IVF-PQ oracle (tests/ivfpq_ref.py).  Every result is
checked by ivfpq_check under its derived per-query tolerance, and every search asserts the list-scan plan the library
reports: (4, sub-quantisers per CTA, CTAs per cluster, candidate warps)."""
import types

import numpy as np
import pytest

from oracle import knn_ref

import ivfpq_ref

pytestmark = pytest.mark.gpu

SMEM_BUDGET = 200 * 1024


def expected_plan(M, k):
    """Restatement of pq_plan (knn_ivfpq.cu): the smallest cluster of 1, 2, 4 CTAs whose table share plus candidate
    lists leaves at least 4 warps within 200 KiB, else the one with the most warps."""
    pitch = (M + 15) // 16 * 16
    best = None
    for cs in (1, 2, 4):
        mc = ((pitch + cs - 1) // cs + 15) // 16 * 16
        for w in (8, 4, 2, 1):
            if mc * 1024 + 2 * (cs - 1) * 256 * 4 + w * k * 8 <= SMEM_BUDGET:
                if best is None or w > best[3]:
                    best = (4, mc, cs, w)
                break
        if best is not None and best[3] >= 4:
            break
    return best


def _build(C, cb, codes, lists, by_residual, nprobe=1, **kw):
    import clip_retrieval_b200 as m

    nlist, d = C.shape
    idx = m.B200IVFPQIndex(d, nlist, cb.shape[0], C, cb, by_residual=by_residual, **kw)
    idx.add_codes(codes, lists)
    idx.nprobe = nprobe
    return idx


def _search_check(idx, Q, C, cb, codes, lists, k, nprobe, by_residual, reconstruct=False, **kw):
    idx.nprobe = nprobe
    if reconstruct:
        D, I, R = idx.search_and_reconstruct(Q, k)
    else:
        D, I = idx.search(Q, k)
        R = None
    assert idx.last_scan_plan() == expected_plan(cb.shape[0], k), (idx.last_scan_plan(), expected_plan(cb.shape[0], k))
    ok, msg, n = ivfpq_ref.ivfpq_check(D, I, Q, C, cb, codes, lists, k, nprobe, by_residual, **kw)
    assert ok, msg
    assert n >= 1
    return D, I, R


SHAPES = [(40, 5), (64, 8), (64, 64), (128, 16), (512, 64), (768, 12), (768, 48), (768, 96), (768, 128), (768, 192),
          (768, 256), (1024, 128)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("by_residual", [True, False])
@pytest.mark.parametrize("d,M", SHAPES)
def test_ivfpq_shapes_k_and_nprobe(d, M, by_residual):
    nlist, n = 16, 2500
    C, cb, codes, lists, _ = ivfpq_ref.make_index(n, d, nlist, M, seed=d + M, by_residual=by_residual, niter=1)
    Q = np.random.default_rng(d * M).standard_normal((5, d)).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    idx = _build(C, cb, codes, lists, by_residual)
    assert idx.M == M and idx.d == d and idx.nlist == nlist and idx.ntotal == n
    for nprobe, ks in ((1, (1, 40)), (7, (40, 1024, 3000)), (nlist, (3000, 8192))):
        for k in ks:
            D, I, R = _search_check(idx, Q, C, cb, codes, lists, k, nprobe, by_residual, reconstruct=(k == 40))
            if k > n:   # more results than rows: padding
                assert (I[:, n:] == -1).all() and (D[:, n:] == knn_ref.NEG).all()
            if R is not None:
                # decoded rows: codeword + centroid in fp32, bit for bit
                sel = I >= 0
                want = ivfpq_ref.reconstruct(C, cb, codes[I[sel]], lists[I[sel]], by_residual)
                assert np.array_equal(R[sel], want)
                assert np.isnan(R[~sel]).all()
    # nprobe = nlist is the exhaustive ADC ranking
    idx.nprobe = nlist
    D, I = idx.search(Q, 40)
    S = ivfpq_ref.adc_scores_f64(Q.astype(np.float64), C, cb, codes, lists, by_residual)
    ok, msg, _ = knn_ref.check_topk(D, I, S, 40, tol=2 * ivfpq_ref.score_error_bound(
        Q.astype(np.float64), C, cb, codes, lists, by_residual).max())
    assert ok, msg


def test_every_cluster_split_is_reached():
    plans = {expected_plan(M, k)[2] for _, M in SHAPES for k in (1, 40, 1024, 3000, 8192)}
    assert plans == {1, 2, 4}


@pytest.mark.timeout(600)
def test_list_shapes_and_query_batches():
    """Empty lists, 1- to 7-row lists and one list holding 60 % of the rows; nq crosses the 256-query batch."""
    d, M, nlist = 64, 16, 24
    rng = np.random.default_rng(7)
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.2).astype(np.float32)
    sizes = np.zeros(nlist, np.int64)
    sizes[1:8] = np.arange(1, 8)          # lists 1..7 hold 1..7 rows; lists 8..10 and 0 stay empty
    sizes[11:] = 120
    sizes[12] = int(0.6 * (sizes.sum() - sizes[12]) / 0.4)   # 60 % of all rows
    lists = np.repeat(np.arange(nlist), sizes)
    perm = rng.permutation(lists.size)
    lists = lists[perm]
    codes = rng.integers(0, 256, (lists.size, M), dtype=np.uint8)
    idx = _build(C, cb, codes, lists, True)
    sz, _ = idx.invlists()
    assert np.array_equal(sz, sizes) and sizes[12] >= 0.6 * sizes.sum() - 1
    for nq in (256, 257):
        Q = rng.standard_normal((nq, d)).astype(np.float32)
        for nprobe, k in ((1, 10), (3, 40), (nlist, 100)):
            _search_check(idx, Q, C, cb, codes, lists, k, nprobe, True)


def _dyadic_index(rng, d, M, nlist, n, dup_lists=False):
    """Values on a 1/64 grid small enough that every fp32 sum is exact: scores are exact in any order."""
    C = (rng.integers(-8, 9, (nlist, d)) / 64.0).astype(np.float32)
    if dup_lists:
        C[1] = C[0]
    cb = (rng.integers(-8, 9, (M, 256, d // M)) / 64.0).astype(np.float32)
    lists = rng.integers(0, nlist, n)
    codes = rng.integers(0, 256, (n, M), dtype=np.uint8)
    return C, cb, codes, lists


@pytest.mark.timeout(300)
def test_ties_come_back_by_ascending_id():
    """Duplicate codes in one list; two lists with identical centroids holding identical codes; a k-th boundary that
    cuts a tie group.  Dyadic values make the fp32 scores exact, so ids must equal the restatement exactly."""
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(11)
    d, M, nlist, n = 64, 8, 6, 3000
    C, cb, codes, lists = _dyadic_index(rng, d, M, nlist, n, dup_lists=True)
    codes[100:400] = codes[100]            # a tie group of 300 rows ...
    lists[100:250] = 0                     # ... half of it in list 0
    lists[250:400] = 1                     # ... half in list 1, whose centroid equals list 0's
    Q = (rng.integers(-8, 9, (4, d)) / 8.0).astype(np.float32)
    Q[:, :] = np.where(np.arange(d) % 2 == 0, Q, 0)
    for by_residual in (True, False):
        idx = _build(C, cb, codes, lists, by_residual)
        for k in (37, 150, 1000):
            for nprobe in (2, nlist):
                idx.nprobe = nprobe
                D, I = idx.search(Q, k)
                Do, Io, _ = ivfpq_ref.ivfpq_search(Q, C, cb, codes, lists, k, nprobe, by_residual)
                assert np.array_equal(I, Io) and np.array_equal(D, Do)
                for q in range(4):
                    tie = (D[q][:-1] == D[q][1:]) & (I[q][1:] >= 0)
                    assert (I[q][:-1][tie] < I[q][1:][tie]).all()
        # the tie group is cut by k: the lowest ids of the group must be the ones returned
        S = ivfpq_ref.adc_scores_f64(Q.astype(np.float64), C, cb, codes, lists, by_residual)
        idx.nprobe = nlist
        for q in range(4):
            s = S[q, 100]
            above = int((S[q] > s).sum())
            k = above + 7
            D, I = idx.search(Q[q:q + 1], k)
            group = np.nonzero(S[q] == s)[0]
            assert np.array_equal(np.sort(I[0, above:]), group[:7])
    assert isinstance(idx, m.B200IVFPQIndex)


@pytest.mark.timeout(300)
def test_range_search_is_strictly_greater():
    rng = np.random.default_rng(5)
    d, M, nlist, n = 32, 4, 5, 2000
    C, cb, codes, lists = _dyadic_index(rng, d, M, nlist, n)
    Q = (rng.integers(-8, 9, (2, d)) / 8.0).astype(np.float32)
    for by_residual in (True, False):
        idx = _build(C, cb, codes, lists, by_residual)
        S = ivfpq_ref.adc_scores_f64(Q.astype(np.float64), C, cb, codes, lists, by_residual)
        for nprobe in (2, nlist):
            idx.nprobe = nprobe
            for q in range(2):
                probes = np.argsort(-(Q[q].astype(np.float64) @ C.T.astype(np.float64)), kind="stable")[:nprobe]
                rows = np.nonzero(np.isin(lists, probes))[0]
                thr = float(np.sort(S[q, rows])[rows.size // 2])   # a row scores exactly the threshold
                assert (S[q, rows] == thr).any()
                lims, D, I = idx.range_search(Q[q:q + 1], thr)
                want = rows[S[q, rows] > thr]
                assert np.array_equal(I, np.sort(want))
                assert np.array_equal(D, S[q, I].astype(np.float32))


@pytest.mark.timeout(300)
def test_serving_shapes_graph_replay_and_batch_rows():
    """nq 1..4 replayed from the CUDA graph equals the eager search bit for bit (with a pre-transform set, so the
    captured launches include it), and nq = 1 equals row 0 of a batch."""
    import torch

    d, M, nlist = 128, 32, 12
    C, cb, codes, lists, _ = ivfpq_ref.make_index(4000, d, nlist, M, seed=9, niter=1)
    A = np.linalg.qr(np.random.default_rng(2).standard_normal((d, d)))[0].astype(np.float32)
    b = np.random.default_rng(3).standard_normal(d).astype(np.float32) * 0.01
    idx = _build(C, cb, codes, lists, True, nprobe=5)
    idx.set_pretransform(A, b)
    Q = np.random.default_rng(4).standard_normal((8, d)).astype(np.float32)
    qd = torch.from_numpy(Q).cuda()
    for nq in (1, 2, 3, 4):
        for k in (10, 40):
            D0, I0, R0 = (t.cpu().numpy() for t in idx.search_device(qd[:nq], k, reconstruct=True))   # eager
            ok, msg, _ = ivfpq_ref.ivfpq_check(D0, I0, Q[:nq], C, cb, codes, lists, k, 5, True, A=A, b=b)
            assert ok, msg
            for _ in range(2):   # graph capture, then replay
                D1, I1, R1 = (t.cpu().numpy() for t in idx.search_device(qd[:nq], k, reconstruct=True))
                assert np.array_equal(D0, D1) and np.array_equal(I0, I1) and np.array_equal(R0, R1, equal_nan=True)
    Db, Ib = idx.search(Q, 40)
    D1, I1 = idx.search(Q[:1], 40)
    assert np.array_equal(D1[0], Db[0]) and np.array_equal(I1[0], Ib[0])


@pytest.mark.timeout(300)
def test_reconstruct_with_opq_and_non_orthonormal_matrix():
    import clip_retrieval_b200 as m

    d, M, nlist = 96, 24, 8
    C, cb, codes, lists, _ = ivfpq_ref.make_index(3000, d, nlist, M, seed=21, niter=1)
    A = np.linalg.qr(np.random.default_rng(1).standard_normal((d, d)))[0].astype(np.float32)
    idx = _build(C, cb, codes, lists, True, nprobe=3)
    idx.set_pretransform(A)
    assert idx.d == d
    Q = np.random.default_rng(8).standard_normal((4, d)).astype(np.float32)
    D, I, R = idx.search_and_reconstruct(Q, 50)
    ok, msg, _ = ivfpq_ref.ivfpq_check(D, I, Q, C, cb, codes, lists, 50, 3, True, A=A)
    assert ok, msg
    sel = I >= 0
    y = ivfpq_ref.reconstruct(C, cb, codes[I[sel]], lists[I[sel]], True).astype(np.float64)
    want = y @ A.astype(np.float64)                          # A^T y, row form
    # a d-term fp32 dot product per output: |err| <= gamma_d * sum_j |A_ji y_j|
    bound = ivfpq_ref.gamma(d) * (np.abs(y) @ np.abs(A.astype(np.float64)))
    assert (np.abs(R[sel] - want) <= bound + 1e-30).all()
    r = idx.reconstruct(int(I[0, 0]))
    assert np.array_equal(r, R[0, 0])
    assert np.isnan(idx.reconstruct(-1)).all()
    # a matrix whose rows are not orthonormal: search works, reconstruct refuses
    idx.set_pretransform(A * 1.01)
    D2, I2 = idx.search(Q, 50)
    ok, msg, _ = ivfpq_ref.ivfpq_check(D2, I2, Q, C, cb, codes, lists, 50, 3, True, A=A * 1.01)
    assert ok, msg
    with pytest.raises(m.B200Error, match="orthonormal"):
        idx.search_and_reconstruct(Q, 5)
    with pytest.raises(m.B200Error, match="orthonormal"):
        idx.reconstruct(0)
    with pytest.raises(NotImplementedError, match="encoder"):
        idx.add(np.zeros((2, d), np.float32))
    with pytest.raises(m.B200Error, match="UNSUPPORTED|add_codes|encoder"):
        m._lib.check(m.lib.b200_index_add_f32(idx._h, np.zeros((1, d), np.float32).ctypes.data, 1, 0), "add_f32")


@pytest.mark.timeout(300)
def test_abi_input_checks():
    import clip_retrieval_b200 as m

    import ctypes

    C = np.zeros((4, 40), np.float32)
    cb = np.zeros((3, 256, 13), np.float32)
    h = ctypes.c_void_p()
    assert m.lib.b200_index_create_ivfpq(40, 4, 3, 1, C.ctypes.data, cb.ctypes.data, 0, ctypes.byref(h)) != 0
    assert b"divide" in m.lib.b200_last_error() and not h
    assert m.lib.b200_index_create_ivfpq(40, 4, 0, 1, C.ctypes.data, cb.ctypes.data, 0, ctypes.byref(h)) != 0
    with pytest.raises(ValueError, match="divide"):
        m.B200IVFPQIndex(40, 4, 3, C, cb)
    with pytest.raises(m.B200Error, match="multiple of 8"):
        m.B200IVFPQIndex(36, 4, 4, np.zeros((4, 36), np.float32), np.zeros((4, 256, 9), np.float32))
    idx = m.B200IVFPQIndex(40, 4, 5, C, np.zeros((5, 256, 8), np.float32))
    with pytest.raises(m.B200Error, match="list 4 of 4"):
        idx.add_codes(np.zeros((2, 5), np.uint8), [0, 4])
    assert m.B200IVFFlatIndex(40, 4, C).d == 40 and int(m.lib.b200_index_pq_m(m.B200IVFFlatIndex(40, 4, C)._h)) == 0


@pytest.mark.timeout(600)
def test_load_index_reads_ivfpq_files(tmp_path):
    import clip_retrieval_b200 as m
    from clip_retrieval_b200 import faiss_io

    d, M, nlist = 64, 16, 10
    C, cb, codes, lists, _ = ivfpq_ref.make_index(3000, d, nlist, M, seed=31, niter=1)
    Q = np.random.default_rng(6).standard_normal((5, d)).astype(np.float32)
    direct = _build(C, cb, codes, lists, True, nprobe=4)
    Dd, Id, Rd = direct.search_and_reconstruct(Q, 40)
    p = str(tmp_path / "image.index")
    faiss_io.write_ivfpq(p, C, cb, codes, lists, nprobe=4)
    idx = m.load_index(p)   # ids of the file are in list order: an id-mapped wrapper around a B200IVFPQIndex
    assert idx.nprobe == 4 and idx.M == M and idx.ntotal == 3000 and idx.nlist == nlist
    D, I, R = idx.search_and_reconstruct(Q, 40)
    assert np.array_equal(D, Dd) and np.array_equal(I, Id) and np.array_equal(R, Rd, equal_nan=True)
    folder = tmp_path / "idx"
    folder.mkdir()
    faiss_io.write_ivfpq(str(folder / "populated.index"), C, cb, codes, lists, nprobe=4, hnsw=True, sparse_sizes=True)
    D2, I2 = m.load_index(str(folder)).search(Q, 40)
    assert np.array_equal(D2, Dd) and np.array_equal(I2, Id)
    # transform + HNSW quantiser + IDMap: ids map on the host, queries go through A
    A = np.linalg.qr(np.random.default_rng(9).standard_normal((d, d)))[0].astype(np.float32)
    ids = np.arange(3000, dtype=np.int64) * 5 + 7
    faiss_io.write_ivfpq(p, C, cb, codes, lists, nprobe=4, transform=(A, None), hnsw=True, id_map=ids)
    loaded = m.load_index(p)
    direct.set_pretransform(A)
    Dt, It = direct.search(Q, 40)
    D3, I3 = loaded.search(Q, 40)
    assert loaded.nprobe == 4 and np.array_equal(D3, Dt) and np.array_equal(I3, ids[It])
    ok, msg, _ = ivfpq_ref.ivfpq_check(Dt, It, Q, C, cb, codes, lists, 40, 4, True, A=A)
    assert ok, msg


@pytest.mark.timeout(300)
def test_two_shards_merge_to_the_single_index():
    import torch
    import clip_retrieval_b200 as m

    d, M, nlist, n = 128, 16, 12, 6000
    C, cb, codes, lists, _ = ivfpq_ref.make_index(n, d, nlist, M, seed=41, niter=1)
    Q = np.random.default_rng(2).standard_normal((6, d)).astype(np.float32)
    full = _build(C, cb, codes, lists, True, nprobe=5)
    D, I = full.search(Q, 100)
    half = n // 2
    a = _build(C, cb, codes[:half], lists[:half], True, nprobe=5)
    b = _build(C, cb, codes[half:], lists[half:], True, nprobe=5)
    b.id_base = half
    qd = torch.from_numpy(Q).cuda()
    Da, Ia = a.search_device(qd, 100)
    Db, Ib = b.search_device(qd, 100)
    Dm, Im = m.merge_shard_results(torch.stack([Da, Db]), torch.stack([Ia, Ib]), 100)
    assert np.array_equal(Dm.cpu().numpy(), D) and np.array_equal(Im.cpu().numpy(), I)


@pytest.mark.timeout(300)
def test_service_query_over_an_ivfpq_resource():
    import clip_retrieval_b200 as m

    d, M, nlist = 64, 8, 8
    C, cb, codes, lists, _ = ivfpq_ref.make_index(3000, d, nlist, M, seed=51, niter=1)
    idx = _build(C, cb, codes, lists, True, nprobe=3)
    q = np.random.default_rng(1).standard_normal((1, d)).astype(np.float32)
    q /= np.linalg.norm(q)
    res = m.ClipResource(types.SimpleNamespace(device="cuda:0"), image_index=idx)
    svc = m.B200KnnService({"img": res})
    out = svc.query(embedding_input=q, num_images=40, num_result_ids=40, deduplicate=False)
    D, I, _ = idx.search_and_reconstruct(q, 40)
    assert [o["id"] for o in out] == I[0][I[0] >= 0].tolist()
    np.testing.assert_array_equal(np.array([o["similarity"] for o in out], np.float32), D[0][I[0] >= 0])
    dedup = svc.query(embedding_input=q, num_images=40, num_result_ids=40, deduplicate=True)
    assert set(o["id"] for o in dedup) <= set(I[0].tolist()) and len(dedup) >= 1


@pytest.mark.timeout(900)
def test_serving_scale():
    """4M rows, nlist 16384, M 64 (d 768), nprobe 32: nq 1000 and nq 1, 8 queries checked on their probed lists."""
    import clip_retrieval_b200 as m

    d, M, nlist, n, nprobe, k = 768, 64, 16384, 4_000_000, 32, 40
    rng = np.random.default_rng(123)
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.05).astype(np.float32)
    lists = rng.integers(0, nlist, n)
    idx = m.B200IVFPQIndex(d, nlist, M, C, cb)
    codes = np.empty((n, M), np.uint8)
    step = 1 << 20
    for s in range(0, n, step):
        codes[s:s + step] = rng.integers(0, 256, (min(step, n - s), M), dtype=np.uint8)
        idx.add_codes(codes[s:s + step], lists[s:s + step])
    idx.nprobe = nprobe
    Q = rng.standard_normal((1000, d)).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    D, I = idx.search(Q, k)
    assert idx.last_scan_plan() == expected_plan(M, k)
    sel = np.arange(0, 1000, 125)
    ok, msg, nchk = ivfpq_ref.ivfpq_check(D[sel], I[sel], Q[sel], C, cb, codes, lists, k, nprobe, True)
    assert ok and nchk >= 6, msg
    D1, I1 = idx.search(Q[:1], k)
    assert np.array_equal(D1[0], D[0]) and np.array_equal(I1[0], I[0])
