"""The fp64 oracle of PCA / ZCA / approximate PCA (tests/pca_oracle.py) against the reference's suites (T/nodes/learning/PCASuite.scala,
ZCAWhiteningSuite.scala) and against the algebra the device relies on.  No GPU."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import pca_oracle as po  # noqa: E402


def _gauss(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32).astype(np.float64)


def test_known_answer_transform():
    """PCASuite "PCA matrix transformation": pcaMat^T x, exact."""
    P = np.array([[1, 2], [3, 4], [5, 6], [7, 8]], dtype=np.float64)
    one = np.arange(12, dtype=np.float64).reshape(4, 3).T
    assert np.array_equal(one @ P, [[102, 120], [118, 140], [134, 160]])
    assert np.array_equal(np.ones((8, 4)) @ P, np.tile([16.0, 20.0], (8, 1)))


def test_pca_estimation_and_distributed():
    """PCASuite "PCA Estimation" and "Covariance Matrix of Distributed PCA should match local one"."""
    X = _gauss(1000, 10, 0)
    P = po.compute_pca(X, 5)
    assert po.off_diagonal_cov(X @ P) < 1e-4
    assert np.abs(po.distributed_pca(np.array_split(X, 4), 5) - P).max() < 1e-4


def test_eigh_route_equals_svd_route():
    for n, d, dims in ((1000, 10, 5), (3000, 130, 80), (50, 120, 30)):
        X = po.planted(n, d, dims, np.random.default_rng(n + d))
        Pe, lam = po.compute_pca_eigh(X, dims)
        assert np.abs(Pe - po.compute_pca(X, dims)).max() < 1e-9
        assert np.abs(lam[:dims] - po.singular_values_sq(X)[:dims]).max() <= 1e-10 * lam[0]


def test_sign_convention_ties_keep_plus():
    P = np.array([[1.0, -2.0, 2.0], [-1.0, 1.0, -2.0]])
    out = po.sign_convention(P)
    assert np.array_equal(out[:, 0], [1.0, -1.0])          # max == max|.|: kept
    assert np.array_equal(out[:, 1], [2.0, -1.0])          # flipped
    assert np.array_equal(out[:, 2], [2.0, -2.0])          # tie between +2 and -2: kept


def test_shard_sums_with_global_mean_give_the_covariance():
    X = _gauss(1001, 40, 1) + 5.0
    mu = X.mean(0)
    shards = [X[:0], X[:7], X[7:500], X[500:]]
    G = sum((s - mu).T @ (s - mu) for s in shards)
    ref = (X - mu).T @ (X - mu)
    assert np.abs(G - ref).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("n,l,shards", [(500, 15, None), (2001, 40, [(0, 3), (3, 1000), (1000, 2001)])])
def test_shifted_cholqr3_equals_householder(n, l, shards):
    Y = _gauss(n, l, n) @ np.diag(np.logspace(0, -6, l))
    Q = po.shifted_cholqr3(Y, shards)
    H = po.householder_q(Y)
    S = np.sign(np.sum(Q * H, 0))
    assert np.abs(Q - H * S).max() < 1e-9
    assert np.abs(Q.T @ Q - np.eye(l)).max() < 1e-12


def test_shifted_cholqr3_on_an_exactly_rank_3_matrix():
    rng = np.random.default_rng(3)
    Y = rng.standard_normal((200, 3)) @ rng.standard_normal((3, 15))
    Q = po.shifted_cholqr3(Y)
    H = po.householder_q(Y)
    assert np.isfinite(Q).all()
    assert np.abs(Q.T @ Q - np.eye(15)).max() < 1e-6
    assert np.linalg.norm(Y - Q @ (Q.T @ Y)) < 1e-10 * np.linalg.norm(Y)
    S = np.sign(np.sum(Q[:, :3] * H[:, :3], 0))           # the leading columns span Y[:, :3] in both
    assert np.abs(Q[:, :3] - H[:, :3] * S).max() < 1e-8


def test_sketch_bound_grid():
    """PCASuite "Sketch algorithm should produce a valid sketch of the matrix" (HMT 1.9) over its (p, k, q) grid."""
    A = _gauss(200, 100, 4)
    s = np.linalg.svd(A, compute_uv=False)
    for p in range(5, 11):
        for k in (1, 5, 10, 20):
            for q in (1, 2, 5, 10, 20):
                Q = po.approximate_q(A, po.omega(100, k + p, p * 100 + k * 10 + q), q)
                assert np.linalg.norm(A - Q @ (Q.T @ A)) < (1 + 9 * np.sqrt(k + p) * 100) * s[k]


def test_approximate_pca_suite_assertions():
    """PCASuite: approximate singular values within mre 0.05, approximate off-diagonal covariance < 0.1; CholeskyQR3 in place of
    Householder gives the same components."""
    A = _gauss(200, 100, 5)
    om = po.omega(100, 15, 0)
    Pa = po.approximate_pca(A, om, 10, 10)
    Pe = po.compute_pca(A, 10)
    sa, se = np.linalg.svd(A @ Pa, compute_uv=False), np.linalg.svd(A @ Pe, compute_uv=False)
    assert np.mean(np.abs(sa - se) / se) < 0.05
    assert po.off_diagonal_cov(A @ Pa) < 0.1
    assert np.abs(po.approximate_pca(A, om, 10, 10, po.shifted_cholqr3) - Pa).max() < 1e-8


def test_zca_suite():
    """ZCAWhiteningSuite: eps 1e-12 whitens to < 1e-4; eps 0.1 to < 0.1 but not < 1e-4."""
    X = _gauss(10000, 10, 6)

    def dev(eps):
        W, mu = po.zca_fit(X, eps)
        return np.abs(np.cov(po.zca_apply(X, W, mu), rowvar=False) - np.eye(10)).max()

    assert dev(1e-12) < 1e-4
    assert dev(0.1) < 0.1 and not dev(0.1) < 1e-4


def test_zca_whitener_from_covariance_eigenpairs():
    """The device's route: V diag(w) V^T = M^T M with M = diag(sqrt(w)) V^T from eigh of the centred covariance."""
    X = _gauss(500, 108, 7)
    X = X - X.mean(1, keepdims=True)                       # rows sum to zero: a null direction
    mu = X.mean(0)
    lam, V = np.linalg.eigh((X - mu).T @ (X - mu))
    w = (np.maximum(lam, 0) / (X.shape[0] - 1) + 1e-5) ** -0.5
    M = np.sqrt(w)[:, None] * V.T
    W, mr = po.zca_fit(X, 1e-5)
    assert np.linalg.norm(M.T @ M - W) / np.linalg.norm(W) < 1e-9


def test_column_pca_selection():
    """PCASuite "small n small d" / "big n big d dense column pca" through the node's host-only optimize."""
    import keystone_b200 as ks
    for n, d, expect in ((1000, 1000, ks.LocalColumnPCAEstimator), (100000, 10000, ks.DistributedColumnPCAEstimator)):
        sample = [np.zeros((d, 10), dtype=np.float32)] * 16
        per = {i: n // (10 * 16) for i in range(16)}
        chosen = ks.ColumnPCAEstimator(100, num_machines=16).optimize(sample, per)
        assert type(chosen) is expect
    args = (960, 1000, 100, 1.0, 16, 3.8e-4, 2.9e-1, 1.32)
    assert ks.PCAEstimator(100).cost(*args) == po.pca_cost(*args)
    assert ks.DistributedPCAEstimator(100).cost(*args) == po.distributed_pca_cost(*args)


def test_node_argument_checks():
    import keystone_b200 as ks
    with pytest.raises(ValueError):
        ks.PCAEstimator(0)
    with pytest.raises(ValueError):
        ks.ZCAWhitenerEstimator(-0.5)
    with pytest.raises(ValueError):
        ks.ZCAWhitenerEstimator(float("nan"))
    with pytest.raises(ValueError):
        ks.ApproximatePCAEstimator(5, q=-1)
    with pytest.raises(ValueError):
        ks.ApproximatePCAEstimator(5, p=-1)
    assert np.array_equal(ks.ApproximatePCAEstimator.omega(7, 3, 4), po.omega(7, 3, 4))
