"""OPQ training on the GPU (b200_opq_train_f32 and its two kernel-level steps) against tests/opq_ref.py."""
import ctypes as C

import numpy as np
import pytest

import ivfpq_ref
import opq_ref as R
import pq_train_ref as P

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24


def _gamma(k):
    return k * U32 / (1 - k * U32)


def _cross(X, codes, cb):
    import torch
    from clip_retrieval_b200._lib import lib, check

    n, d_in = X.shape
    M, _, dsub = cb.shape
    Xd = torch.from_numpy(np.ascontiguousarray(X, np.float32)).cuda()
    cd = torch.from_numpy(np.ascontiguousarray(codes, np.uint8)).cuda()
    cbd = torch.from_numpy(np.ascontiguousarray(cb, np.float32)).cuda()
    G = torch.empty((M * dsub, d_in), dtype=torch.float32, device="cuda")
    check(lib.b200_opq_cross_f32_device(Xd.data_ptr(), n, d_in, cd.data_ptr(), cbd.data_ptr(), M * dsub, M,
                                        G.data_ptr(), 0, torch.cuda.current_stream().cuda_stream), "opq_cross")
    return G.cpu().numpy()


def _polar(G):
    import torch
    from clip_retrieval_b200._lib import lib, check

    Gd = torch.from_numpy(np.ascontiguousarray(G, np.float32)).cuda()
    A = torch.empty_like(Gd)
    check(lib.b200_opq_polar_f32_device(Gd.data_ptr(), G.shape[0], G.shape[1], A.data_ptr(), 0,
                                        torch.cuda.current_stream().cuda_stream), "opq_polar")
    return A.cpu().numpy()


def test_cross_step_exact_on_dyadic_data():
    rng = np.random.default_rng(0)
    n, d_in, M, dsub = 3000, 80, 6, 8   # ragged row chunk, ragged tiles on both sides
    X = rng.integers(-8, 9, (n, d_in)).astype(np.float32) / 16
    cb = (rng.integers(-8, 9, (M, 256, dsub)) / 16).astype(np.float32)
    codes = rng.integers(0, 256, (n, M)).astype(np.uint8)
    G = _cross(X, codes, cb)
    ref = R.decode(codes, cb).astype(np.float64).T @ X.astype(np.float64)
    assert np.array_equal(G.astype(np.float64), ref)


def test_cross_step_bounded_and_deterministic():
    """Within a 1024-row chunk each entry is a sequential fma chain: |err| <= gamma_1024 sum |y||x|; the chunk partials
    (at most ceil(n / 1024)) are then added in order, which adds gamma_{chunks - 1} times the sum of their magnitudes,
    itself at most (1 + gamma_1024) sum |y||x|."""
    rng = np.random.default_rng(1)
    n, d_in, M = 5000, 96, 12
    X = rng.standard_normal((n, d_in)).astype(np.float32)
    cb = rng.standard_normal((M, 256, 8)).astype(np.float32)
    codes = rng.integers(0, 256, (n, M)).astype(np.uint8)
    G = _cross(X, codes, cb)
    Y = R.decode(codes, cb).astype(np.float64)
    ref = Y.T @ X.astype(np.float64)
    mag = np.abs(Y).T @ np.abs(X.astype(np.float64))
    chunks = -(-n // 1024)
    bound = (_gamma(1024) + _gamma(chunks - 1) * (1 + _gamma(1024))) * mag
    assert (np.abs(G - ref) <= bound).all(), float((np.abs(G - ref) / bound).max())
    assert np.array_equal(G.view(np.uint32), _cross(X, codes, cb).view(np.uint32))


def test_polar_step():
    rng = np.random.default_rng(2)
    d_out, d_in = 48, 64
    U = R.polar(rng.standard_normal((d_out, d_out)))
    V = R.polar(rng.standard_normal((d_out, d_in)))
    G = (U * np.logspace(0, 3, d_out)) @ V
    G32 = G.astype(np.float32)
    A = _polar(G32)
    assert np.abs(A - R.polar(G32.astype(np.float64))).max() <= 1e-6
    # rank-deficient G: the rows are still orthonormal
    Gr = ((rng.standard_normal((d_out, 5)) @ rng.standard_normal((5, d_in)))).astype(np.float32)
    Ar = _polar(Gr).astype(np.float64)
    assert np.abs(Ar @ Ar.T - np.eye(d_out)).max() <= 1e-6


def test_initial_rotation_matches_the_restatement():
    import clip_retrieval_b200 as m

    X = np.random.default_rng(3).standard_normal((512, 64)).astype(np.float32)
    A, obj = m.train_opq(X, 8, d_out=48, niter=0)
    assert obj.shape == (0,)
    assert np.abs(A - R.initial_rotation(48, 64, 1234)).max() <= 1e-6
    with pytest.raises(ValueError):
        m.train_opq(X, 8, d_out=72)


def test_one_iteration_from_the_seeded_picks():
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(4)
    n, d, M = 2048, 32, 4
    X = (rng.standard_normal((n, d)) * np.linspace(2, 0.2, d)).astype(np.float32)
    A0, _ = m.train_opq(X, M, niter=0)
    A1, obj = m.train_opq(X, M, niter=1, niter_pq_0=0)
    # the device's codes: those of the seeded picks of x A0^T (fp32), under the gap / bound rule of check_encode
    xp = (X.astype(np.float64) @ A0.astype(np.float64).T)
    xp32 = xp.astype(np.float32)
    x_err = ivfpq_ref.pretransform_error_bound(X, A0) + U32 * np.abs(xp)
    cb = np.ascontiguousarray(xp32.reshape(n, M, d // M)[P.sample_picks(n, 256, 1234)].transpose(1, 0, 2))
    idx = m.B200IVFPQIndex(d, 1, M, np.zeros((1, d), np.float32), cb, by_residual=False)
    idx.set_pretransform(A0)
    codes, lists = idx.encode(X)
    ok, msg, _ = P.check_encode(codes, lists, xp, np.zeros((1, d), np.float32), cb, False, x_err=x_err)
    assert ok, msg
    Y = R.decode(codes, cb).astype(np.float64)
    assert np.abs(A1 - R.polar(Y.T @ X.astype(np.float64))).max() <= 1e-5
    assert abs(obj[0] - ((xp - Y) ** 2).sum() / n) <= 1e-5 * obj[0]


def _anisotropic(n, d, seed):
    rng = np.random.default_rng(seed)
    Q = R.polar(rng.standard_normal((d, d)))
    return ((rng.standard_normal((n, d)) * np.exp(-np.arange(d) / (d / 8))) @ Q.T).astype(np.float32)


# The restatement run on the CPU in float32 and in float64 (tests/opq_ref.py, this data, 10 iterations, niter_pq_0 10,
# niter_pq 4) gives per-iteration objectives that differ by at most SMALL_SPREAD relative; the device may sit anywhere
# in that spread on either side of the float64 run, so the tolerance is twice it.
SMALL_SPREAD = 2.4e-3   # measured: 2.396e-3, at iteration 8


def test_full_training_at_small_size():
    import clip_retrieval_b200 as m

    X = _anisotropic(4096, 64, 5)
    A, obj = m.train_opq(X, 8, niter=10, niter_pq_0=10)
    _, o64, _, _, _ = R.train_opq(X, 8, niter=10, niter_pq=4, niter_pq_0=10)
    assert np.all(np.abs(obj - o64) <= 2 * SMALL_SPREAD * o64), (obj, o64)
    assert np.abs(A.astype(np.float64) @ A.T - np.eye(64)).max() <= 1e-5


# PQ error of OPQ over plain PQ (same trainer, as many Lloyd iterations) on the small anisotropic data, as the
# restatement measures it: 0.1819 / 0.7020 = 0.259, a 74 % cut.  At real size the device must keep at least half that cut.
SMALL_RATIO = 1 - (1 - 0.259) / 2


def test_full_training_at_real_size():
    import torch
    import clip_retrieval_b200 as m

    n, d, M = 65536, 768, 64
    X = torch.from_numpy(_anisotropic(n, d, 6)).cuda()
    A, obj = m.train_opq(X, M)
    A2, obj2 = m.train_opq(X, M)
    assert np.array_equal(A.view(np.uint32), A2.view(np.uint32)) and np.array_equal(obj, obj2)
    assert obj[-1] < obj[0]
    idx = m.B200IVFPQIndex(d, 1, M, np.zeros((1, d), np.float32), np.zeros((M, 256, d // M), np.float32))
    idx.set_pretransform(A)
    from clip_retrieval_b200._lib import lib
    info = np.zeros(8, np.int32)
    lib.b200_index_get_quantizer(idx._h, None, None, None, None, info.ctypes.data)
    assert info[3] == 1
    cb, _ = m.train_pq(X, M, niter=40 + 49 * 4)
    Xn = X.cpu().numpy().astype(np.float64)
    codes, _ = m.B200IVFPQIndex(d, 1, M, np.zeros((1, d), np.float32), cb, by_residual=False).encode(X)
    pq_err = ((Xn - R.decode(codes.cpu().numpy(), cb)) ** 2).sum() / n
    print("real size: OPQ objective %.6g -> %.6g, plain PQ %.6g, ratio %.4f" % (obj[0], obj[-1], pq_err, obj[-1] / pq_err))
    assert obj[-1] <= SMALL_RATIO * pq_err


def test_build_ivfpq_index_with_opq_end_to_end():
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(7)
    n, d, M, nlist = 20000, 64, 8, 32
    X = _anisotropic(n, d, 8)
    idx = m.build_ivfpq_index(X, nlist, M, opq_dim=48, opq_niter=8, nprobe=4)
    assert idx.d == 64
    info = np.zeros(8, np.int32)
    from clip_retrieval_b200._lib import lib
    cent = np.empty((nlist, 48), np.float32)
    cb = np.empty((M, 256, 6), np.float32)
    A = np.empty((48, 64), np.float32)
    lib.b200_index_get_quantizer(idx._h, cent.ctypes.data, cb.ctypes.data, A.ctypes.data, None, info.ctypes.data)
    assert list(info[:7]) == [nlist, M, 1, 1, 0, 48, 64]
    sizes, ids = idx.invlists()
    codes_slot = np.empty((n, M), np.uint8)
    lib.b200_index_copy_rows(idx._h, 0, n, codes_slot.ctypes.data, None)
    codes = np.empty_like(codes_slot)
    codes[ids] = codes_slot
    lists = np.empty(n, np.int64)
    lists[ids] = np.repeat(np.arange(nlist), sizes)
    Q = X[rng.choice(n, 16, replace=False)] + 0.01 * rng.standard_normal((16, d)).astype(np.float32)
    D, I = idx.search(Q, 10)
    ok, msg, checked = ivfpq_ref.ivfpq_check(D, I, Q, cent, cb, codes, lists, 10, 4, True, A=A)
    assert ok and checked >= 12, (msg, checked)


def test_training_phases_and_cross_refusal():
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200._lib import lib

    X = _anisotropic(2048, 32, 9)
    A, obj = m.train_opq(X, 4, niter=3, niter_pq_0=2)
    A2, obj2, ph = m.train_opq(X, 4, niter=3, niter_pq_0=2, phases=True)
    assert np.array_equal(A, A2) and np.array_equal(obj, obj2)   # timing adds synchronisations, not arithmetic
    assert set(ph) == {"rotate", "pq", "cross", "svd"} and all(v > 0 for v in ph.values())
    buf = torch.zeros(64, device="cuda")
    rc = lib.b200_opq_cross_f32_device(buf.data_ptr(), 65537, 8, buf.data_ptr(), buf.data_ptr(), 8, 1, buf.data_ptr(), 0,
                                       None)
    assert rc != 0 and b"65536" in lib.b200_last_error()


def test_pretransform_rows_fp32_fp16_and_any_width():
    import torch
    import clip_retrieval_b200 as m

    rng = np.random.default_rng(10)
    n, d_in = 3000, 64
    X = rng.standard_normal((n, d_in)).astype(np.float16)
    for d_out in (48, 36):
        A = rng.standard_normal((d_out, d_in)).astype(np.float32)
        b = rng.standard_normal(d_out).astype(np.float32)
        Y = m.index.pretransform_rows(X, A, b, chunk=1000).cpu().numpy()
        ref = X.astype(np.float64) @ A.astype(np.float64).T + b
        bound = ivfpq_ref.pretransform_error_bound(X.astype(np.float32), A, b)
        assert (np.abs(Y - ref) <= bound).all()
        Yh = m.index.pretransform_rows(torch.from_numpy(X).cuda(), A, b, dtype="float16")
        assert Yh.dtype == torch.float16 and np.array_equal(Yh.cpu().numpy(), Y.astype(np.float16))
    # the same bits as the encoder's pre-transform (the residual output of an index without residuals)
    A = rng.standard_normal((48, d_in)).astype(np.float32)
    idx = m.B200IVFPQIndex(48, 1, 6, np.zeros((1, 48), np.float32), np.zeros((6, 256, 8), np.float32), by_residual=False)
    idx.set_pretransform(A)
    xt = torch.from_numpy(X.astype(np.float32)).cuda()
    res = torch.empty((n, 48), device="cuda")
    from clip_retrieval_b200._lib import lib, check
    check(lib.b200_index_encode_device(idx._h, xt.data_ptr(), n, None, res.data_ptr(), None,
                                       torch.cuda.current_stream().cuda_stream), "encode")
    assert torch.equal(res, m.index.pretransform_rows(xt, A))
