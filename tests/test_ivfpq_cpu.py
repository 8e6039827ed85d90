"""IVF-PQ files and the IVF-PQ oracle, without a GPU.  The reader is round-tripped through faiss_io's own writer of
the layout (UNVERIFIED against FAISS-written files: FAISS cannot be run here)."""
import struct

import numpy as np
import pytest

from clip_retrieval_b200 import faiss_io
from oracle import knn_ref

import ivfpq_ref


def _small(d=32, nlist=6, M=8, n=300, by_residual=True, seed=3):
    C, cb, codes, lists, X = ivfpq_ref.make_index(n, d, nlist, M, seed=seed, by_residual=by_residual, niter=1)
    return C, cb, codes, lists


def _orthonormal(d, seed=0):
    q, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((d, d)))
    return q.astype(np.float32)


def _assert_same(r, C, cb, codes, lists, ids, nprobe, by_residual):
    nlist = C.shape[0]
    order = np.argsort(lists, kind="stable")
    assert r["kind"] == "ivfpq" and r["nlist"] == nlist and r["nprobe"] == nprobe and r["M"] == cb.shape[0]
    assert r["by_residual"] == by_residual and r["ntotal"] == codes.shape[0]
    assert np.array_equal(r["centroids"], C) and np.array_equal(r["codebook"], cb)
    assert np.array_equal(r["list_sizes"], np.bincount(lists, minlength=nlist))
    assert r["codes"].dtype == np.uint8 and np.array_equal(r["codes"], codes[order])
    assert np.array_equal(r["ids"], ids[order])


@pytest.mark.parametrize("by_residual", [True, False])
def test_ivfpq_round_trip(tmp_path, by_residual):
    C, cb, codes, lists = _small(by_residual=by_residual)
    ids = np.arange(codes.shape[0], dtype=np.int64) * 3 + 5
    p = str(tmp_path / "image.index")
    faiss_io.write_ivfpq(p, C, cb, codes, lists, ids=ids, nprobe=4, by_residual=by_residual)
    raw = open(p, "rb").read()
    assert raw[:4] == b"IwPQ"
    r = faiss_io.read_faiss_index(p)
    _assert_same(r, C, cb, codes, lists, ids, 4, by_residual)
    assert r["transform"] is None


def test_ivfpq_hnsw_quantizer_sparse_sizes_and_empty_lists(tmp_path):
    C, cb, codes, lists = _small(nlist=9)
    lists = lists % 4          # lists 4..8 stay empty
    p = str(tmp_path / "image.index")
    faiss_io.write_ivfpq(p, C, cb, codes, lists, nprobe=2, hnsw=True, sparse_sizes=True)
    r = faiss_io.read_faiss_index(p)
    _assert_same(r, C, cb, codes, lists, np.arange(codes.shape[0]), 2, True)
    assert (r["list_sizes"][4:] == 0).all()
    # the HNSW quantiser is skipped, not served: a top-level HNSW index stays unsupported
    raw = open(p, "rb").read()
    at = raw.index(b"IHNf")
    open(p, "wb").write(raw[at:])
    with pytest.raises(NotImplementedError, match="load_index"):
        faiss_io.read_faiss_index(p)


@pytest.mark.parametrize("tag,bias", [("LTra", True), ("rrot", False)])
def test_ivfpq_pretransform_and_id_map(tmp_path, tag, bias):
    C, cb, codes, lists = _small()
    d = C.shape[1]
    A = _orthonormal(d)
    b = np.linspace(-0.1, 0.1, d).astype(np.float32) if bias else None
    ids = np.arange(codes.shape[0], dtype=np.int64)[::-1] * 2
    p = str(tmp_path / "image.index")
    faiss_io.write_ivfpq(p, C, cb, codes, lists, nprobe=3, transform=(A, b), transform_tag=tag, hnsw=True, id_map=ids)
    raw = open(p, "rb").read()
    assert raw[:4] == b"IxMp" and raw[37:41] == b"IxPT"
    r = faiss_io.read_faiss_index(p)
    _assert_same(r, C, cb, codes, lists, ids, 3, True)
    A2, b2 = r["transform"]
    assert np.array_equal(A2, A) and (b2 is None if b is None else np.array_equal(b2, b))


def test_ivfpq_refusals(tmp_path):
    C, cb, codes, lists = _small()
    p = str(tmp_path / "image.index")
    faiss_io.write_ivfpq(p, C, cb, codes, lists, nbits=4)
    with pytest.raises(NotImplementedError, match="8-bit"):
        faiss_io.read_faiss_index(p)
    faiss_io.write_ivfpq(p, C, cb, codes, lists, code_size=codes.shape[1] + 1)
    with pytest.raises(ValueError, match="code size"):
        faiss_io.read_faiss_index(p)
    # d % M != 0: a PQ of M = 8 over a declared d of 36
    faiss_io.write_ivfpq(p, C, cb, codes, lists, pq_d=36)
    with pytest.raises(ValueError, match="M must divide d"):
        faiss_io.read_faiss_index(p)
    # a chain of two transforms
    faiss_io.write_ivfpq(p, C, cb, codes, lists, transform=(_orthonormal(C.shape[1]), None))
    raw = bytearray(open(p, "rb").read())
    assert raw[:4] == b"IxPT"
    struct.pack_into("<i", raw, 37, 2)
    open(p, "wb").write(bytes(raw))
    with pytest.raises(NotImplementedError, match="load_index"):
        faiss_io.read_faiss_index(p)


def test_oracle_fp32_restatement_within_the_derived_bound():
    for d, M, by_residual in ((32, 8, True), (48, 48, False), (64, 4, True)):
        C, cb, codes, lists, _ = ivfpq_ref.make_index(600, d, 5, M, seed=M, by_residual=by_residual, niter=1)
        Q = np.random.default_rng(1).standard_normal((4, d)).astype(np.float32)
        k = 50
        D, I, _ = ivfpq_ref.ivfpq_search(Q, C, cb, codes, lists, k, 5, by_residual)
        ok, msg, n = ivfpq_ref.ivfpq_check(D, I, Q, C, cb, codes, lists, k, 5, by_residual)
        assert ok and n == 4, msg
        S64 = ivfpq_ref.adc_scores_f64(Q.astype(np.float64), C, cb, codes, lists, by_residual)
        bound = ivfpq_ref.score_error_bound(Q.astype(np.float64), C, cb, codes, lists, by_residual)
        for q in range(4):
            sel = I[q] >= 0
            assert np.all(np.abs(D[q, sel] - S64[q, I[q, sel]]) <= bound[q, I[q, sel]])
        # the bound grows with M: a fixed 2e-6 is not a bound at M = 256
        assert ivfpq_ref.gamma(257) * 1.0 > 1.5e-5


def test_oracle_adc_equals_inner_product_with_the_reconstruction():
    for by_residual in (True, False):
        C, cb, codes, lists, _ = ivfpq_ref.make_index(200, 24, 4, 6, seed=2, by_residual=by_residual, niter=1)
        Q = np.random.default_rng(5).standard_normal((3, 24))
        S = ivfpq_ref.adc_scores_f64(Q, C, cb, codes, lists, by_residual)
        R = ivfpq_ref.reconstruct(C, cb, codes, lists, by_residual).astype(np.float64)
        if by_residual:   # the fp32 add of the reconstruction rounds; compare with the exact sum
            R = cb[np.arange(6)[None, :], codes.astype(np.int64)].reshape(200, 24).astype(np.float64) + C[lists].astype(np.float64)
        np.testing.assert_allclose(S, Q @ R.T, rtol=0, atol=1e-12)


def test_oracle_encoding_picks_the_nearest_codeword():
    rng = np.random.default_rng(0)
    X = rng.standard_normal((500, 16)).astype(np.float32)
    cb = ivfpq_ref.train_pq(X, 4, niter=2)
    codes = ivfpq_ref.encode(X, cb)
    for m in range(4):
        xs = X[:, m * 4:(m + 1) * 4].astype(np.float64)
        d2 = ((xs[:, None, :] - cb[m][None].astype(np.float64)) ** 2).sum(-1)
        assert np.array_equal(codes[:, m], np.argmin(d2, axis=1))
    assert knn_ref.NEG == np.float32(-3.4028234663852886e38)
