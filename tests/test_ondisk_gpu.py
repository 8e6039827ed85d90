"""IVF-PQ with lists in host memory (csrc/knn_ivfpq_stream.cu) against the resident load of the same file: the same
bits for D, I and R of search / search_and_reconstruct / search_device and the same range_search arrays, over the
shapes of test_ivfpq_gpu.py, tie groups, tiny arenas, ids past 2^32, the LAION layout through the service, merged
parts, nprobe changes, two threads and a serving-scale index."""
import os
import threading
import types

import numpy as np
import pytest

import ivfpq_ref

pytestmark = pytest.mark.gpu

SHAPES = [(40, 5), (64, 8), (64, 64), (128, 16), (512, 64), (768, 12), (768, 48), (768, 96), (768, 128), (768, 192),
          (768, 256), (1024, 128)]


def _inner(index):
    return getattr(index, "_index", index)


def _load_pair(folder, arena=None):
    import clip_retrieval_b200 as m

    res = m.load_index(folder, max_device_bytes=1 << 40)
    st = m.load_index(folder, max_device_bytes=0)
    assert not _inner(res).streamed and _inner(st).streamed
    if arena is not None:
        _inner(st).set_stream_arena(arena)
    return res, st


def _same(res, st, Q, k, nprobe, device=True, ranges=True):
    import torch

    _inner(res).nprobe = nprobe
    _inner(st).nprobe = nprobe
    D0, I0, R0 = res.search_and_reconstruct(Q, k)
    D1, I1, R1 = st.search_and_reconstruct(Q, k)
    assert np.array_equal(D0, D1) and np.array_equal(I0, I1) and np.array_equal(R0, R1, equal_nan=True)
    D2, I2 = st.search(Q, k)
    assert np.array_equal(D2, D0) and np.array_equal(I2, I0)
    if device:
        qd = torch.from_numpy(Q).cuda()
        a = [t.cpu().numpy() for t in res.search_device(qd, k, reconstruct=True)]
        b = [t.cpu().numpy() for t in st.search_device(qd, k, reconstruct=True)]
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2], equal_nan=True)
        assert np.array_equal(b[1], I0)
        c = [t.cpu().numpy() for t in st.search_device(qd, k)]
        assert np.array_equal(c[0], D0) and np.array_equal(c[1], I0)
    if ranges:
        for q in range(min(2, Q.shape[0])):
            live = D0[q][I0[q] >= 0]
            thr = float(live[len(live) // 2]) if len(live) else 0.0
            la, Da, Ia = res.range_search(Q[q:q + 1], thr)
            lb, Db, Ib = st.range_search(Q[q:q + 1], thr)
            assert np.array_equal(la, lb) and np.array_equal(Da, Db) and np.array_equal(Ia, Ib)
    return D0, I0


def _write(tmp_path, name, C, cb, codes, lists, ids, by_residual=True, **kw):
    from clip_retrieval_b200 import faiss_io

    folder = str(tmp_path / name)
    faiss_io.write_ivfpq_ondisk(folder, C, cb, codes, lists, ids=ids, nprobe=1, by_residual=by_residual, **kw)
    return folder


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("by_residual", [True, False])
@pytest.mark.parametrize("d,M", SHAPES)
def test_streamed_equals_resident(tmp_path, d, M, by_residual):
    nlist, n = 16, 2500
    C, cb, codes, lists, _ = ivfpq_ref.make_index(n, d, nlist, M, seed=d + M, by_residual=by_residual, niter=1)
    ids = (np.random.default_rng(M).permutation(n).astype(np.int64) * 3 + (5 << 32))   # file ids past 2^32
    folder = _write(tmp_path, "idx", C, cb, codes, lists, ids, by_residual)
    res, st = _load_pair(folder)
    Q = np.random.default_rng(d * M).standard_normal((300, d)).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    for nprobe, k in ((1, 1), (1, 40), (7, 40), (7, 3000), (nlist, 3000)):
        for nq in (1, 7):
            D, I = _same(res, st, Q[:nq], k, nprobe, ranges=(k == 40))
            assert (I[I >= 0] >= (5 << 32)).all()
            plan = _inner(res).last_scan_plan()   # both residencies launch the same list scan
            assert plan[0] == 4 and _inner(st).last_scan_plan() == plan, (plan, _inner(st).last_scan_plan())
    _same(res, st, Q, 40, 7, device=False, ranges=False)         # 300 queries: beyond one pass
    # an arena of the least size: passes alternate between the two arenas
    _inner(st).set_stream_arena(0)
    _same(res, st, Q[:7], 40, 7)
    st.search(Q[:7], 40)
    assert _inner(st).last_stream_stats()["passes"] >= 2


@pytest.mark.timeout(600)
def test_ties_across_lists_and_tiny_arena(tmp_path):
    """Dyadic values: exact ties, two lists with the same centroid and the same codes, a k that cuts a tie group."""
    rng = np.random.default_rng(11)
    d, M, nlist, n = 64, 8, 6, 3000
    C = (rng.integers(-8, 9, (nlist, d)) / 64.0).astype(np.float32)
    C[1] = C[0]
    cb = (rng.integers(-8, 9, (M, 256, d // M)) / 64.0).astype(np.float32)
    lists = rng.integers(0, nlist, n)
    codes = rng.integers(0, 256, (n, M), dtype=np.uint8)
    codes[100:400] = codes[100]
    lists[100:250] = 0
    lists[250:400] = 1
    Q = (rng.integers(-8, 9, (9, d)) / 8.0).astype(np.float32)
    for by_residual in (True, False):
        folder = _write(tmp_path, "t%d" % by_residual, C, cb, codes, lists, np.arange(n, dtype=np.int64) * 7 + 1,
                        by_residual)
        res, st = _load_pair(folder, arena=0)
        for k in (37, 150, 1000):
            for nprobe in (1, 2, nlist):
                D, I = _same(res, st, Q, k, nprobe, device=(k == 150))
                tie = (D[:, :-1] == D[:, 1:]) & (I[:, 1:] >= 0)
                assert tie.any()


@pytest.mark.timeout(600)
def test_laion_layout_through_the_service(tmp_path):
    """IxPT(LTra) -> IwPQ with an IHNf quantiser and on-disk lists, loaded from its folder: the service returns the
    file's ids, streamed and resident (the resident index is id-mapped: its search_device maps ids on the device)."""
    import clip_retrieval_b200 as m

    d, M, nlist, n = 64, 16, 12, 4000
    C, cb, codes, lists, _ = ivfpq_ref.make_index(n, d, nlist, M, seed=61, niter=1)
    A = np.linalg.qr(np.random.default_rng(3).standard_normal((d, d)))[0].astype(np.float32)
    ids = np.random.default_rng(4).permutation(n).astype(np.int64) + (1 << 33)
    folder = _write(tmp_path, "laion", C, cb, codes, lists, ids, transform=(A, None), hnsw=True,
                    recorded_dir="/data/merge")
    q = np.random.default_rng(5).standard_normal((1, d)).astype(np.float32)
    q /= np.linalg.norm(q)
    direct = m.B200IVFPQIndex(d, nlist, M, C, cb)
    direct.add_codes(codes, lists)
    direct.set_pretransform(A)
    direct.nprobe = 4
    Dd, Id = direct.search(q, 40)
    for budget in (None, 0):
        idx = m.load_index(folder, max_device_bytes=budget)
        assert _inner(idx).streamed == (budget == 0) and idx.ntotal == n
        _inner(idx).nprobe = 4
        res = m.ClipResource(types.SimpleNamespace(device="cuda:0"), image_index=idx)
        svc = m.B200KnnService({"img": res})
        out = svc.query(embedding_input=q, num_images=40, num_result_ids=40, deduplicate=False)
        assert [o["id"] for o in out] == ids[Id[0][Id[0] >= 0]].tolist()
        np.testing.assert_array_equal(np.array([o["similarity"] for o in out], np.float32), Dd[0][Id[0] >= 0])
        dedup = svc.query(embedding_input=q, num_images=40, num_result_ids=40, deduplicate=True)
        assert set(o["id"] for o in dedup) <= set(ids.tolist()) and len(dedup) >= 1
    st = m.load_index(folder, max_device_bytes=0)
    with pytest.raises(NotImplementedError, match="host memory"):
        st.reconstruct(0)
    sizes, got = st.invlists()
    order = np.argsort(lists, kind="stable")
    assert np.array_equal(sizes, np.bincount(lists, minlength=nlist)) and np.array_equal(got, ids[order])


@pytest.mark.timeout(900)
def test_merged_parts_equal_one_index(tmp_path):
    import clip_retrieval_b200 as m
    from clip_retrieval_b200 import faiss_io

    d, M, nlist, n, nparts = 128, 16, 32, 12000, 3
    rng = np.random.default_rng(7)
    X = rng.standard_normal((n, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    C, cb = m.train_ivfpq(X, nlist, M, niter=4, pq_niter=4)
    enc = m.B200IVFPQIndex(d, nlist, M, C, cb)
    src = tmp_path / "parts"
    src.mkdir()
    bounds = np.linspace(0, n, nparts + 1).astype(int)
    for i in range(nparts):
        codes, lists = enc.encode(X[bounds[i]:bounds[i + 1]])
        faiss_io.write_ivfpq(str(src / ("knn_%d.index" % i)), C, cb, codes, lists, nprobe=8,
                             ids=np.arange(bounds[i], bounds[i + 1], dtype=np.int64))
    m.index_combiner(str(src), str(tmp_path / "merged"))
    st = m.load_index(str(tmp_path / "merged"), max_device_bytes=0)
    one = m.B200IVFPQIndex(d, nlist, M, C, cb)
    one.add_codes(*one.encode(X))
    one.nprobe = 8
    assert st.nprobe == 8 and st.ntotal == n
    Q = rng.standard_normal((50, d)).astype(np.float32)
    for k in (10, 100):
        D0, I0, R0 = one.search_and_reconstruct(Q, k)
        D1, I1, R1 = st.search_and_reconstruct(Q, k)
        assert np.array_equal(D0, D1) and np.array_equal(I0, I1) and np.array_equal(R0, R1, equal_nan=True)


@pytest.mark.timeout(600)
def test_nprobe_changes_and_two_threads(tmp_path):
    d, M, nlist, n = 128, 32, 24, 20000
    C, cb, codes, lists, _ = ivfpq_ref.make_index(n, d, nlist, M, seed=71, niter=1)
    folder = _write(tmp_path, "th", C, cb, codes, lists, np.arange(n, dtype=np.int64)[::-1].copy())
    res, st = _load_pair(folder, arena=1 << 16)
    Q = np.random.default_rng(8).standard_normal((64, d)).astype(np.float32)
    want = {}
    for nprobe in (3, 11, 1, nlist, 3):
        want[nprobe] = _same(res, st, Q, 40, nprobe, device=False, ranges=False)
    _inner(st).nprobe = 5
    _inner(res).nprobe = 5
    ref = res.search(Q, 40)
    errors = []

    def worker(seed):
        try:
            rng = np.random.default_rng(seed)
            for _ in range(6):
                s = int(rng.integers(0, 60))
                D, I = st.search(Q[s:s + 4], 40)
                if not (np.array_equal(D, ref[0][s:s + 4]) and np.array_equal(I, ref[1][s:s + 4])):
                    errors.append(seed)
        except Exception as e:   # noqa: BLE001  (reported below)
            errors.append(repr(e))

    th = [threading.Thread(target=worker, args=(s,)) for s in (1, 2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


@pytest.mark.timeout(1800)
def test_streamed_serving_scale(tmp_path):
    """4M rows, nlist 16384, M 64 (d 768), nprobe 32, as test_serving_scale: streamed equals resident for nq 1000
    and nq 1."""
    from clip_retrieval_b200 import faiss_io

    d, M, nlist, n, nprobe, k = 768, 64, 16384, 4_000_000, 32, 40
    rng = np.random.default_rng(123)
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.05).astype(np.float32)
    lists = rng.integers(0, nlist, n)
    codes = rng.integers(0, 256, (n, M), dtype=np.uint8)
    folder = str(tmp_path / "scale")
    faiss_io.write_ivfpq_ondisk(folder, C, cb, codes, lists, nprobe=nprobe)
    del codes
    res, st = _load_pair(folder)
    Q = rng.standard_normal((1000, d)).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    D0, I0 = res.search(Q, k)
    D1, I1 = st.search(Q, k)
    assert np.array_equal(D0, D1) and np.array_equal(I0, I1)
    D2, I2 = st.search(Q[:1], k)
    assert np.array_equal(D2[0], D0[0]) and np.array_equal(I2[0], I0[0])
    assert os.path.getsize(os.path.join(folder, "merged_index.ivfdata")) >= n * (M + 8)
