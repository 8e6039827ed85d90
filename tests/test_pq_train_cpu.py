"""Self-checks of the PQ encoding / training oracle (tests/pq_train_ref.py), without a GPU."""
import numpy as np

from oracle.kmeans_ref import initial_picks

import pq_train_ref as P


def _dyadic(rng, shape, lim=8, den=64.0):
    return (rng.integers(-lim, lim + 1, shape) / den).astype(np.float32)


def test_encoder_matches_float64_brute_force_on_exact_data():
    rng = np.random.default_rng(0)
    for d, M, nlist in ((64, 8, 5), (32, 32, 3), (48, 1, 4)):
        X, C, cb = _dyadic(rng, (300, d)), _dyadic(rng, (nlist, d)), _dyadic(rng, (M, 256, d // M))
        for by_residual in (True, False):
            codes, lists = P.encode(X, C, cb, by_residual)
            want_l = np.array([max(range(nlist), key=lambda l: (float(np.dot(x.astype(np.float64), C[l])), -l))
                               for x in X])
            assert np.array_equal(lists, want_l)
            R = X.astype(np.float64) - (C[lists] if by_residual else 0)
            dsub = d // M
            for i in range(0, 300, 37):
                for m in range(M):
                    dist = ((R[i, m * dsub:(m + 1) * dsub][None] - cb[m].astype(np.float64)) ** 2).sum(1)
                    assert codes[i, m] == int(np.flatnonzero(dist == dist.min())[0])
            ok, msg, _ = P.check_encode(codes, lists, X, C, cb, by_residual)
            assert ok, msg


def test_ties_go_to_the_lower_index():
    d, M = 16, 4
    C = np.zeros((3, d), np.float32)
    C[1] = C[2] = 0.5
    cb = np.zeros((M, 256, d // M), np.float32)
    cb[:, 7] = 0.25
    cb[:, 3] = 0.25                     # codewords 3 and 7 equal: 3 must win
    X = np.full((2, d), 0.5, np.float32)
    codes, lists = P.encode(X, C, cb, False)
    assert (lists == 1).all() and (codes == 3).all()


def test_a_wrong_choice_fails_the_tolerant_check():
    rng = np.random.default_rng(1)
    X = rng.standard_normal((50, 32)).astype(np.float32)
    C = rng.standard_normal((6, 32)).astype(np.float32)
    cb = rng.standard_normal((4, 256, 8)).astype(np.float32)
    codes, lists = P.encode(X, C, cb, True)
    assert P.check_encode(codes, lists, X, C, cb, True)[0]
    bad = codes.copy()
    bad[3, 2] ^= 1
    assert not P.check_encode(bad, lists, X, C, cb, True)[0]
    worst = np.argmin(X.astype(np.float64) @ C.astype(np.float64).T, axis=1)
    assert not P.check_encode(codes, worst, X, C, cb, True)[0]


def test_trainer_recovers_planted_sub_vector_centres():
    rng = np.random.default_rng(2)
    M, dsub, n = 2, 4, 256 * 12
    centres = rng.standard_normal((M, 256, dsub)).astype(np.float32) * 4
    owner = np.stack([np.arange(n) * 256 // n for _ in range(M)], axis=1)   # rows grouped by centre: one pick each
    X = np.concatenate([centres[m][owner[:, m]] for m in range(M)], axis=1)
    X = (X + 1e-3 * rng.standard_normal(X.shape)).astype(np.float32)
    cb, sizes, codes = P.train_pq(X, M, niter=3, seed=5)
    assert (sizes == n // 256).all()
    for m in range(M):
        assert np.abs(cb[m] - centres[m]).max() < 5e-3
        assert np.array_equal(codes[:, m], owner[:, m])


def test_split_rule_on_duplicated_rows():
    """Fewer distinct sub-vectors than codewords: duplicate picks leave codewords empty, and each is re-seeded from
    the largest one of its m with the +-1/1024 perturbation, sizes halving."""
    rng = np.random.default_rng(3)
    base = rng.standard_normal((3, 8)).astype(np.float32)
    X = np.repeat(base, [150, 90, 60], axis=0)
    cb, sizes, _ = P.train_pq(X, 2, niter=1, seed=4)
    picks = initial_picks(300, 256, 4)
    assert len(np.unique(X[picks], axis=0)) == 3
    assert sizes.sum(axis=1).tolist() == [300, 300]
    # after one update + split round the codewords of every m are perturbed copies of the three updated means, each
    # split taking the (then) largest: ratios to the source alternate 1 + eps / 1 - eps by column on the first split
    for m in range(2):
        v = np.zeros(4, np.float32)
        for _ in range(150):                         # the update: fp32 sum in row order, times fp32 1/count
            v = v + X[0, m * 4:(m + 1) * 4]
        v = v * (np.float32(1) / np.float32(150))
        assert len(np.unique(cb[m], axis=0)) > 3
        ratio = cb[m].astype(np.float64) / v.astype(np.float64)
        near = np.abs(ratio - 1).max(axis=1) < 0.05        # descendants of the largest cluster
        assert near.sum() > 3
    assert np.array_equal(P.sample_picks(1000, 65536, 1), np.arange(1000))
