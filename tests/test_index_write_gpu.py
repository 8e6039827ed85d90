"""faiss_io.write_index and clip_index: files byte-identical to the fixture writers', read back by load_index with the
in-memory index's results, streamed with bounded host memory."""
import os
import tracemalloc

import numpy as np
import pytest

from clip_retrieval_b200 import faiss_io

pytestmark = pytest.mark.gpu


def _bytes(p):
    with open(p, "rb") as f:
        return f.read()


def _ivf_assign(idx):
    sizes, ids = idx.invlists()
    lists = np.empty(len(ids), np.int64)
    lists[ids] = np.repeat(np.arange(len(sizes)), sizes)
    return sizes, ids, lists


def _same_results(a, b, Q, k):
    Da, Ia, Ra = a.search_and_reconstruct(Q, k)
    Db, Ib, Rb = b.search_and_reconstruct(Q, k)
    assert np.array_equal(Da, Db)
    tie = np.zeros_like(Da, dtype=bool)
    tie[:, 1:] |= Da[:, 1:] == Da[:, :-1]
    tie[:, :-1] |= Da[:, :-1] == Da[:, 1:]
    assert np.array_equal(Ia[~tie], Ib[~tie])
    for q in range(Q.shape[0]):   # a loaded file breaks exact ties by file position: same ids per tied score
        for s in np.unique(Da[q][tie[q]]):
            assert sorted(Ia[q][Da[q] == s]) == sorted(Ib[q][Db[q] == s])
    assert np.array_equal(Ra[~tie], Rb[~tie])


def test_byte_identity_with_the_fixture_writers(tmp_path):
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(0)
    n, d, nlist, M = 3000, 64, 16, 8
    X = rng.standard_normal((n, d)).astype(np.float16)
    a, b = str(tmp_path / "a.index"), str(tmp_path / "b.index")
    # flat fp16
    flat = m.B200FlatIndex(d)
    flat.add(X)
    m.write_index(flat, a)
    faiss_io.write_flat(b, X, fp16=True)
    assert _bytes(a) == _bytes(b)
    # IVF-Flat with fp16-representable centroids; within a list, ascending insertion id
    cent = X[rng.choice(n, nlist, replace=False)].astype(np.float32)
    ivf = m.B200IVFFlatIndex(d, nlist, cent)
    ivf.add(X)
    ivf.nprobe = 3
    m.write_index(ivf, a)
    _, _, lists = _ivf_assign(ivf)
    faiss_io.write_ivfflat(b, cent, X, lists, nprobe=3, fp16=True)
    assert _bytes(a) == _bytes(b)
    # IVF-PQ with / without residuals, with / without a pre-transform
    C = rng.standard_normal((nlist, 48)).astype(np.float32)
    cb = rng.standard_normal((M, 256, 6)).astype(np.float32)
    codes = rng.integers(0, 256, (n, M)).astype(np.uint8)
    lists = rng.integers(0, nlist, n)
    A = np.linalg.qr(rng.standard_normal((d, 48)))[0].T.astype(np.float32)
    for by_residual in (True, False):
        for transform in (None, (A, None), (A, rng.standard_normal(48).astype(np.float32))):
            pq = m.B200IVFPQIndex(48, nlist, M, C, cb, by_residual=by_residual)
            if transform is not None:
                pq.set_pretransform(*transform)
            pq.add_codes(codes[:1000], lists[:1000])
            pq.add_codes(codes[1000:], lists[1000:])
            pq.nprobe = 5
            m.write_index(pq, a, chunk_bytes=1 << 12)
            faiss_io.write_ivfpq(b, C, cb, codes, lists, nprobe=5, by_residual=by_residual, transform=transform)
            assert _bytes(a) == _bytes(b)
    # an id map, as load_index returns it.  A loaded file's rows are inserted in list order, so the written file numbers
    # them 0..n-1 in list order: the fixture is made in that canonical order (same index, same search results).
    id_map = rng.permutation(10 * n)[:n].astype(np.int64)
    order = np.argsort(lists, kind="stable")
    codes, lists, id_map = codes[order], lists[order], id_map[order]
    faiss_io.write_ivfpq(b, C, cb, codes, lists, nprobe=2, transform=(A, None), id_map=id_map)
    m.write_index(m.load_index(b), a)
    assert _bytes(a) == _bytes(b)
    faiss_io.write_flat(b, X, fp16=True, id_map=id_map)
    m.write_index(m.load_index(b), a)
    assert _bytes(a) == _bytes(b)


def test_refusals(tmp_path):
    import clip_retrieval_b200 as m

    with pytest.raises(TypeError):
        m.write_index(object(), str(tmp_path / "x.index"))
    flat = m.B200FlatIndex(16)
    flat.add(np.ones((4, 16), np.float32))
    flat.id_base = 100
    with pytest.raises(ValueError, match="id_base"):
        m.write_index(flat, str(tmp_path / "x.index"))


def test_round_trip(tmp_path):
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(1)
    n, d = 20000, 64
    X = rng.standard_normal((n, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    Q = X[rng.choice(n, 8, replace=False)] + 0.05 * rng.standard_normal((8, d)).astype(np.float32)
    p = str(tmp_path / "r.index")
    for idx in (m.build_ivf_index(X, 32, nprobe=4),
                m.build_ivfpq_index(X, 32, 8, nprobe=4),
                m.build_ivfpq_index(X, 32, 8, nprobe=4, opq_dim=64, opq_niter=4)):
        m.write_index(idx, p)
        _same_results(idx, m.load_index(p), Q, 20)
    flat = m.B200FlatIndex(d)
    flat.add(X)
    m.write_index(flat, p)
    _same_results(flat, m.load_index(p), Q, 20)


def test_write_streams_with_bounded_host_memory(tmp_path):
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(2)
    n, d, M, nlist = 2_000_000, 64, 16, 1024
    idx = m.B200IVFPQIndex(d, nlist, M, rng.standard_normal((nlist, d)).astype(np.float32),
                           rng.standard_normal((M, 256, d // M)).astype(np.float32))
    for s in range(0, n, 1 << 20):
        e = min(n, s + (1 << 20))
        idx.add_codes(rng.integers(0, 256, (e - s, M)).astype(np.uint8), rng.integers(0, nlist, e - s))
    idx.finalize()
    chunk = 1 << 22
    p = str(tmp_path / "big.index")
    tracemalloc.start()
    m.write_index(idx, p, chunk_bytes=chunk)
    _, peak = tracemalloc.get_traced_memory()
    tracemalloc.stop()
    assert os.path.getsize(p) > n * (M + 8)
    assert peak < 3 * chunk, peak


def _shards(root, rng, name, sizes, d, centers):
    os.makedirs(os.path.join(root, name))
    for i, s in enumerate(sizes):
        x = centers[rng.integers(0, len(centers), s)] + 0.3 * rng.standard_normal((s, d))
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        np.save(os.path.join(root, name, "%s_%02d.npy" % (name, i)), x.astype(np.float16))


@pytest.mark.parametrize("key", ["SQfp16", "IVF16,Flat", "OPQ8_64,IVF16_HNSW32,PQ8x8", None])
def test_clip_index_end_to_end(tmp_path, key):
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(3)
    d = 64
    centers = rng.standard_normal((40, d))
    emb = str(tmp_path / "emb")
    _shards(emb, rng, "img_emb", [5000, 0, 4000, 3000], d, centers)
    _shards(emb, rng, "text_emb", [6000, 6500], d, centers)
    os.makedirs(os.path.join(emb, "metadata"))
    with open(os.path.join(emb, "metadata", "metadata_0.parquet"), "wb") as f:
        f.write(b"PAR1 not really")
    out = str(tmp_path / "index")
    m.clip_index(emb, out, index_key=key)
    assert _bytes(os.path.join(out, "metadata", "metadata_0.parquet")) == b"PAR1 not really"
    for name, sub in (("image", "img_emb"), ("text", "text_emb")):
        loaded = m.load_index(os.path.join(out, name + ".index"))
        built = m.build_index(os.path.join(emb, sub), index_key=key)
        assert loaded.ntotal == built.ntotal == (12000 if name == "image" else 12500)
        if key is None:   # 12 000 rows fit the 4G budget as fp16: IVF{2^round(log2(4 sqrt(12000)))},SQfp16
            assert loaded.nlist == 512
        if key != "SQfp16":
            assert loaded.nprobe == built.nprobe == m.default_nprobe(loaded.nlist)
        Q = np.load(os.path.join(emb, sub, sorted(os.listdir(os.path.join(emb, sub)))[0]))[:6].astype(np.float32)
        _same_results(built, loaded, Q, 10)


def test_clip_index_nprobe_and_width_refusal(tmp_path):
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(4)
    emb = str(tmp_path / "emb")
    _shards(emb, rng, "img_emb", [3000], 64, rng.standard_normal((10, 64)))
    os.makedirs(os.path.join(emb, "metadata"))
    out = str(tmp_path / "index")
    m.clip_index(emb, out, index_key="IVF32,PQ8x8", nprobe=7)
    assert not os.path.exists(os.path.join(out, "text.index"))
    assert m.load_index(os.path.join(out, "image.index")).nprobe == 7
    with pytest.raises(ValueError, match="multiple of 8"):
        m.build_index(os.path.join(emb, "img_emb"), index_key="OPQ4_36,IVF16,PQ4x8")
