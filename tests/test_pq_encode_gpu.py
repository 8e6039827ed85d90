"""IVF-PQ encoding and PQ training on the GPU (csrc/pq_encode.cu) against tests/pq_train_ref.py.  On dyadic data every
fp32 product and sum is exact, so codes, lists and trained codebooks must equal the oracle bit for bit; on random
data each choice must lie within the derived per-element bound of the best one."""
import numpy as np
import pytest

import ivfpq_ref
import pq_train_ref as P
from test_ivfpq_gpu import SHAPES

pytestmark = pytest.mark.gpu


def _dyadic(rng, shape, lim=8, den=64.0):
    return (rng.integers(-lim, lim + 1, shape) / den).astype(np.float32)


def _index(C, cb, by_residual=True):
    import clip_retrieval_b200 as m

    return m.B200IVFPQIndex(C.shape[1], C.shape[0], cb.shape[0], C, cb, by_residual=by_residual)


def _residuals_device(idx, X):
    import torch
    import clip_retrieval_b200 as m

    x = torch.from_numpy(np.ascontiguousarray(X, np.float32)).cuda()
    r = torch.empty((X.shape[0], idx._d_code), dtype=torch.float32, device=x.device)
    m._lib.check(m.lib.b200_index_encode_device(idx._h, x.data_ptr(), X.shape[0], None, r.data_ptr(), None, None), "encode")
    torch.cuda.synchronize()
    return r.cpu().numpy()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("by_residual", [True, False])
@pytest.mark.parametrize("d,M", SHAPES + [(256, 256), (2048, 1)])
def test_exact_encode(d, M, by_residual):
    rng = np.random.default_rng(d * 7 + M)
    nlist, n = 37, 700
    C, cb, X = _dyadic(rng, (nlist, d)), _dyadic(rng, (M, 256, d // M)), _dyadic(rng, (n, d))
    C[5] = C[3]                                          # two equal centroids: list 3 must win over 5
    X[:20] = C[3] * 4                                    # rows that mostly choose the tied lists
    cb[:, 200] = cb[:, 17]                               # two equal codewords per m: 17 must win over 200
    X[20:40] = np.tile(cb[:, 17].reshape(-1), (20, 1))  # without residuals: at distance 0 from both
    idx = _index(C, cb, by_residual)
    codes, lists = idx.encode(X)
    want_c, want_l = P.encode(X, C, cb, by_residual)
    assert (want_l[:20] == 3).mean() > 0.5 and np.array_equal(lists, want_l)
    assert (codes != 200).all()
    if not by_residual:   # distance 0: the lowest codeword equal to codeword 17 (small dsub repeats codewords)
        first = [int(np.flatnonzero((cb[m] == cb[m, 17]).all(axis=1))[0]) for m in range(M)]
        assert (codes[20:40] == np.array(first, np.uint8)[None]).all()
    assert codes.dtype == np.uint8 and codes.shape == (n, M) and lists.dtype == np.int64
    assert np.array_equal(codes, want_c)
    want_r = P.residuals(X, C, want_l, by_residual)
    assert np.array_equal(_residuals_device(idx, X), want_r)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("d,M,nlist", [(768, 64, 500), (128, 16, 64), (256, 256, 40)])
def test_tolerant_encode_on_random_unit_rows(d, M, nlist):
    rng = np.random.default_rng(d + M)
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    X = rng.standard_normal((3000, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.05).astype(np.float32)
    for by_residual in (True, False):
        codes, lists = _index(C, cb, by_residual).encode(X)
        ok, msg, close = P.check_encode(codes, lists, X, C, cb, by_residual)
        assert ok, msg
        print("d %d M %d nlist %d by_residual %d: %d of %d rows decided inside a bound" % (
            d, M, nlist, by_residual, close, X.shape[0]))


@pytest.mark.timeout(600)
def test_coarse_tile_edges():
    rng = np.random.default_rng(3)
    d, M = 64, 8
    cb = _dyadic(rng, (M, 256, d // M))
    for nlist in (1, 63, 64, 65, 127, 128, 129, 4097):
        C = _dyadic(rng, (nlist, d))
        idx = _index(C, cb)
        for n in (1, 63, 65, 127, 129, 1000):
            X = _dyadic(rng, (n, d))
            codes, lists = idx.encode(X)
            want_c, want_l = P.encode(X, C, cb, True)
            assert np.array_equal(lists, want_l), (nlist, n)
            assert np.array_equal(codes, want_c), (nlist, n)
    # the best list in the last tile only, and in the first only
    C = _dyadic(rng, (4097, d))
    C[4096] = 1.0
    X = np.abs(_dyadic(rng, (5, d))) + 1 / 64
    _, lists = _index(C, cb).encode(X)
    assert (lists == 4096).all()


@pytest.mark.timeout(600)
def test_pretransform_and_loaded_opq_file(tmp_path):
    import clip_retrieval_b200 as m
    from clip_retrieval_b200 import faiss_io

    rng = np.random.default_rng(8)
    d, d_in, M, nlist = 96, 128, 24, 30
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.05).astype(np.float32)
    A = np.linalg.qr(rng.standard_normal((d_in, d_in)))[0][:d].astype(np.float32)
    b = (rng.standard_normal(d) * 0.01).astype(np.float32)
    X = rng.standard_normal((2000, d_in)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    Xt = ivfpq_ref.transform_f64(X, A, b)
    err = ivfpq_ref.pretransform_error_bound(X, A, b)
    idx = _index(C, cb)
    idx.set_pretransform(A, b)
    assert idx.d == d_in
    codes, lists = idx.encode(X)
    ok, msg, close = P.check_encode(codes, lists, Xt, C, cb, True, x_err=err)
    assert ok, msg
    print("pre-transform: %d of %d rows decided inside a bound" % (close, X.shape[0]))
    # an OPQ + HNSW + IVF-PQ file (square rotation, as autofaiss writes) encodes the same way
    Aq = np.linalg.qr(rng.standard_normal((d, d)))[0].astype(np.float32)
    p = str(tmp_path / "opq.index")
    codes0 = rng.integers(0, 256, (100, M), dtype=np.uint8)
    faiss_io.write_ivfpq(p, C, cb, codes0, np.sort(rng.integers(0, nlist, 100)), nprobe=3, transform=(Aq, None),
                         hnsw=True)
    loaded = m.load_index(p)
    assert isinstance(loaded, m.B200IVFPQIndex) and loaded.d == d
    Xq = X[:, :d].copy()
    codes2, lists2 = loaded.encode(Xq)
    ok, msg, _ = P.check_encode(codes2, lists2, ivfpq_ref.transform_f64(Xq, Aq), C, cb, True,
                                x_err=ivfpq_ref.pretransform_error_bound(Xq, Aq))
    assert ok, msg
    direct = _index(C, cb)
    direct.set_pretransform(Aq)
    c3, l3 = direct.encode(Xq)
    assert np.array_equal(c3, codes2) and np.array_equal(l3, lists2)


def _planted(rng, n, d, M, spread=1e-3):
    """Rows whose every sub-vector sits near one of 256 planted centres, grouped centre after centre so the stride picks
    start one codeword in every group."""
    dsub = d // M
    centres = (rng.standard_normal((M, 256, dsub)) * 2).astype(np.float32)
    for m in range(M):   # centres at least 0.25 apart along their first column
        centres[m, :, 0] = rng.permutation(256) * 0.25
    owner = (np.arange(n) * 256) // n
    X = np.concatenate([centres[m][owner] for m in range(M)], axis=1)
    return (X + spread * rng.standard_normal(X.shape)).astype(np.float32)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("d,M", [(64, 64), (64, 8), (128, 2), (512, 2)])
def test_training_matches_the_oracle(d, M):
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(d + M)
    X = _planted(rng, 256 * 10, d, M)
    cb, sizes = m.train_pq(X, M, niter=4, seed=9)
    want, wsizes, _ = P.train_pq(X, M, 4, seed=9)
    gap, bound = P.codeword_gaps(X, want)
    assert (gap > bound).all()
    np.testing.assert_array_equal(sizes, wsizes)
    np.testing.assert_array_equal(cb, want)
    cb2, sizes2 = m.train_pq(X, M, niter=4, seed=9)            # determinism
    assert np.array_equal(cb, cb2) and np.array_equal(sizes, sizes2)


@pytest.mark.timeout(600)
def test_training_splits_empty_codewords_and_refuses_bad_shapes():
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(4)
    base = _dyadic(rng, (5, 16))
    # 5 distinct sub-vectors per m for 256 codewords; power-of-two counts keep every mean, perturbed copy and distance
    # exact in fp32, so the device's ties (to the lower codeword) are the oracle's
    X = np.repeat(base, [128, 64, 32, 16, 16], axis=0)
    cb, sizes = m.train_pq(X, 4, niter=3, seed=3)
    want, wsizes, _ = P.train_pq(X, 4, 3, seed=3)
    np.testing.assert_array_equal(sizes, wsizes)
    np.testing.assert_array_equal(cb, want)
    with pytest.raises(m.B200Error, match="256"):
        m.train_pq(X[:255], 4)
    with pytest.raises(ValueError, match="divide"):
        m.train_pq(X, 5)
    with pytest.raises(m.B200Error, match="divide"):
        m._lib.check(m.lib.b200_pq_train_f32(X.ctypes.data, 300, 16, 5, 1, 0, X.ctypes.data, None, 0), "pq_train")


@pytest.mark.timeout(600)
def test_determinism_chunks_and_device_input():
    import torch

    rng = np.random.default_rng(6)
    d, M, nlist = 128, 32, 300
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.1).astype(np.float32)
    X = rng.standard_normal((40000, d)).astype(np.float32)
    idx = _index(C, cb)
    codes, lists = idx.encode(X)
    c2, l2 = idx.encode(X, chunk=777)
    assert np.array_equal(codes, c2) and np.array_equal(lists, l2)
    parts = [idx.encode(X[s:s + 9999]) for s in range(0, X.shape[0], 9999)]
    assert np.array_equal(codes, np.concatenate([p[0] for p in parts]))
    assert np.array_equal(lists, np.concatenate([p[1] for p in parts]))
    cd, ld = idx.encode(torch.from_numpy(X).cuda())
    assert cd.is_cuda and cd.dtype == torch.uint8 and np.array_equal(cd.cpu().numpy(), codes)
    assert np.array_equal(ld, lists)
    X16 = X.astype(np.float16)
    c16, l16 = idx.encode(torch.from_numpy(X16).cuda())
    c16h, l16h = idx.encode(X16)
    assert np.array_equal(c16.cpu().numpy(), c16h) and np.array_equal(l16, l16h)
    assert np.array_equal(c16h, idx.encode(X16.astype(np.float32))[0])


def _clustered(rng, n, d, nc, spread=0.35):
    cent = rng.standard_normal((nc, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    X = cent[rng.integers(0, nc, n)] + spread * rng.standard_normal((n, d)).astype(np.float32) / np.sqrt(d)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X.astype(np.float16)


@pytest.mark.timeout(1200)
def test_build_ivfpq_index_end_to_end():
    import clip_retrieval_b200 as m
    from oracle import knn_ref

    rng = np.random.default_rng(12)
    d, nlist, M, n = 768, 256, 64, 200_000
    X = _clustered(rng, n, d, 1000)
    idx = m.build_ivfpq_index(X, nlist, M, niter=4, pq_niter=8, nprobe=16)
    cent, cb = m.train_ivfpq(X, nlist, M, niter=4, pq_niter=8)
    codes, lists = idx.encode(X)
    sizes, _ = idx.invlists()
    assert idx.ntotal == n and np.array_equal(sizes, np.bincount(lists, minlength=nlist))
    Q = X[rng.choice(n, 64, replace=False)].astype(np.float32)
    D, I, R = idx.search_and_reconstruct(Q, 10)
    ok, msg, nchk = ivfpq_ref.ivfpq_check(D, I, Q, cent, cb, codes, lists, 10, 16, True)
    assert ok and nchk >= 32, msg
    flat = m.B200FlatIndex(d)
    flat.add(X)
    _, If = flat.search(Q, 10)
    recall = np.mean([len(set(I[q]) & set(If[q])) / 10 for q in range(Q.shape[0])])
    print("recall@10 against the exact flat search: %.3f" % recall)
    assert recall >= 0.12   # 0.169 measured on an H100 80GB HBM3 (deterministic seeds)
    # decoding then re-encoding gives back the row's code and list on exact data
    rng2 = np.random.default_rng(13)
    Cd, cbd = np.eye(16, 64, dtype=np.float32), _dyadic(rng2, (8, 256, 8))   # lists far apart, small codewords
    e = _index(Cd, cbd)
    Xd = Cd[rng2.integers(0, 16, 500)] + _dyadic(rng2, (500, 64))
    cd, ld = e.encode(Xd)
    e.add_codes(cd, ld)
    e.finalize()
    Rr = np.stack([e.reconstruct(i) for i in range(0, 500, 25)])
    c2, l2 = e.encode(Rr)
    assert np.array_equal(c2, cd[::25]) and np.array_equal(l2, ld[::25])
    assert knn_ref is not None


@pytest.mark.timeout(600)
def test_shards_encoded_against_one_quantiser_merge_to_the_single_index():
    import torch
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(21)
    d, nlist, M, n = 128, 32, 16, 20000
    X = _clustered(rng, n, d, 200)
    cent, cb = m.train_ivfpq(X, nlist, M, niter=3, pq_niter=5)
    full = _index(cent, cb)
    full.add_codes(*full.encode(X))
    full.finalize()
    full.nprobe = 4
    half = n // 2
    shards = []
    for s, e in ((0, half), (half, n)):
        sh = _index(cent, cb)
        sh.add_codes(*sh.encode(X[s:e]))
        sh.finalize()
        sh.nprobe = 4
        sh.id_base = s
        shards.append(sh)
    Q = torch.from_numpy(X[:8].astype(np.float32)).cuda()
    D, I = full.search_device(Q, 50)
    parts = [s.search_device(Q, 50) for s in shards]
    Dm, Im = m.merge_shard_results(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), 50)
    assert torch.equal(Dm, D) and torch.equal(Im, I)


@pytest.mark.timeout(1200)
def test_encode_at_scale_with_bounded_scratch():
    import torch
    import clip_retrieval_b200 as m

    d, M, nlist, n = 768, 64, 16384, 4_000_000
    rng = np.random.default_rng(31)
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.05).astype(np.float32)
    idx = _index(C, cb)
    X = m.index.synth_rows(n, d, m.SynthSpec(seed=5), dtype="float32")
    torch.cuda.synchronize()
    free0, res0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    codes, lists = idx.encode(X, chunk=1 << 20)
    torch.cuda.synchronize()
    free1, res1 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    lib_growth = (free0 - free1) - (res1 - res0)          # what the library kept past the call
    chunk_scratch = (1 << 20) * 4                         # the int32 lists of one chunk (torch)
    assert res1 - res0 <= n * M + chunk_scratch + (64 << 20), (res1 - res0)
    assert lib_growth <= 64 << 20, lib_growth
    sel = np.arange(0, n, n // 8)[:8]
    Xs = X[torch.from_numpy(sel).cuda()].cpu().numpy()
    ok, msg, _ = P.check_encode(codes[torch.from_numpy(sel).cuda()].cpu().numpy(), lists[sel], Xs, C, cb, True)
    assert ok, msg
    assert lists.min() >= 0 and lists.max() < nlist
