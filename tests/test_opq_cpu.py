"""The OPQ restatement (tests/opq_ref.py) checked against itself: its Procrustes step is the optimum of the trace
objective, and its training objective never increases while no codeword is split."""
import numpy as np

import opq_ref as R


def _random_orthogonal_near_identity(rng, k, eps):
    return R.polar(np.eye(k) + eps * rng.standard_normal((k, k)))


def test_procrustes_step_beats_every_perturbation():
    rng = np.random.default_rng(0)
    for d_out, d_in in ((16, 16), (12, 20)):
        G = rng.standard_normal((d_out, d_in))
        A = R.polar(G)
        assert np.allclose(A @ A.T, np.eye(d_out), atol=1e-12)
        best = R.procrustes_objective(A, G)
        for i in range(100):
            eps = 10.0 ** rng.uniform(-4, 0)
            P = A @ _random_orthogonal_near_identity(rng, d_in, eps) if i % 2 else \
                _random_orthogonal_near_identity(rng, d_out, eps) @ A
            assert R.procrustes_objective(P, G) < best


def test_initial_rotation_is_seeded_and_orthonormal():
    A = R.initial_rotation(24, 32, 1234)
    assert np.allclose(A @ A.T, np.eye(24), atol=1e-12)
    assert np.array_equal(A, R.initial_rotation(24, 32, 1234))
    assert not np.allclose(A, R.initial_rotation(24, 32, 1235))
    g = R.gaussian(64, 64, 7).ravel()
    assert abs(g.mean()) < 0.05 and abs(g.std() - 1) < 0.05


def test_objective_never_increases_without_splits():
    rng = np.random.default_rng(3)
    n, d, M = 4096, 16, 4
    X = (rng.standard_normal((n, d)) * np.linspace(3, 0.3, d)).astype(np.float32)
    A, obj, splits, _, _ = R.train_opq(X, M, niter=6, niter_pq=2, niter_pq_0=4)
    assert splits == 0
    assert np.all(np.diff(obj) <= 1e-6 * obj[:-1]), obj
    assert obj[-1] < obj[0]
