"""Gaussian-kernel ridge regression on the host: the fp64 oracle (tests/krr_oracle.py) against the reference's
KernelModelSuite and against the direct solve, the increment form the device fit uses, the two-rank label fold, and argument
checks of the nodes that need no GPU."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import krr_oracle as ko  # noqa: E402

XOR_X = np.array([[-1.0, -1.0], [1.0, 1.0], [-1.0, 1.0], [1.0, -1.0]])
XOR_Y = np.array([[0.0, 1.0], [0.0, 1.0], [1.0, 0.0], [1.0, 0.0]])


@pytest.mark.parametrize("block_size", [4, 2])
def test_xor_known_answer(block_size):
    """T/nodes/learning/KernelModelSuite.scala: gamma 10, lambda 0, 2 epochs, squared error on 3 training points < 1e-4."""
    xs = ko.krr_fit(XOR_X, XOR_Y, 10.0, 0.0, block_size, 2)
    pred = ko.kernel_block_apply(XOR_X[:3], XOR_X, 10.0, xs, block_size)
    assert np.sum((pred - XOR_Y[:3]) ** 2) < 1e-4


def _problem(n=230, d=5, k=3, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    Y = rng.standard_normal((n, k))
    return X, Y


def test_one_block_is_the_direct_solve():
    X, Y = _problem()
    gamma, lam = 0.3, 0.5
    K = ko.gaussian_kernel(X, X, gamma)
    direct = np.linalg.solve(K + lam * np.eye(len(X)), Y)
    xs = ko.krr_fit(X, Y, gamma, lam, 1000, 1)
    assert len(xs) == 1
    assert np.abs(xs[0] - direct).max() < 1e-10


def test_many_epochs_converge_to_the_direct_solve():
    X, Y = _problem()
    gamma, lam = 1.0, 1.0
    direct = np.linalg.solve(ko.gaussian_kernel(X, X, gamma) + lam * np.eye(len(X)), Y)
    W = np.concatenate(ko.krr_fit(X, Y, gamma, lam, 64, 40), 0)
    assert np.abs(W - direct).max() < 1e-8


def _increment_form(X, Y, gamma, lam, bs, epochs, order=None):
    """What the device computes: rhs = Y_B - K_B^T W - lam W_B, dW = (K_BB + lam I) \\ rhs, W_B += dW."""
    n = len(X)
    blocks = ko.block_ranges(n, bs)
    W = np.zeros_like(Y)
    for e in range(epochs):
        for j in (range(len(blocks)) if order is None else order[e]):
            lo, hi = blocks[j]
            KB = ko.gaussian_kernel(X, X[lo:hi], gamma)
            rhs = Y[lo:hi] - KB.T @ W - lam * W[lo:hi]
            W[lo:hi] += np.linalg.solve(KB[lo:hi] + lam * np.eye(hi - lo), rhs)
    return W


@pytest.mark.parametrize("permuted", [False, True])
def test_increment_form_equals_reference_form(permuted):
    X, Y = _problem()                 # 230 rows, block size 64: a 38-row ragged tail
    gamma, lam, bs, epochs = 0.3, 0.5, 64, 3
    nb = len(ko.block_ranges(len(X), bs))
    order = None
    if permuted:
        rng = np.random.Generator(np.random.PCG64(7))
        order = [rng.permutation(nb) for _ in range(epochs)]
    ref = np.concatenate(ko.krr_fit(X, Y, gamma, lam, bs, epochs, order), 0)
    inc = _increment_form(X, Y, gamma, lam, bs, epochs, order)
    assert np.abs(ref - inc).max() < 1e-12


def test_two_shard_label_fold():
    """Rows split over two ranks, a block straddling the split: the sum of the per-rank K_B^T W - Y_B(own rows) is C - Y_B."""
    X, Y = _problem()
    rng = np.random.default_rng(3)
    W = rng.standard_normal(Y.shape)
    split, (lo, hi) = 100, (64, 128)
    KB = ko.gaussian_kernel(X, X[lo:hi], 0.3)
    total = np.zeros((hi - lo, Y.shape[1]))
    for r0, r1 in ((0, split), (split, len(X))):
        part = KB[r0:r1].T @ W[r0:r1]
        f0, f1 = max(lo, r0), min(hi, r1)
        part[f0 - lo:f1 - lo] -= Y[f0:f1]
        total += part
    assert np.allclose(total, KB.T @ W - Y[lo:hi], rtol=0, atol=1e-12)


def test_gaussian_kernel_translation_invariance():
    X, _ = _problem(n=50)
    Z = X[:20] * 0.7
    a = ko.gaussian_kernel(X, Z, 0.2)
    b = ko.gaussian_kernel(X + 3.0, Z + 3.0, 0.2)
    assert np.abs(a - b).max() < 1e-12
    assert np.allclose(np.diag(ko.gaussian_kernel(X, X, 0.2)), 1.0)


def test_diag_block_is_rows_of_the_column_block():
    X, _ = _problem(n=50)
    idx = np.arange(10, 25)
    col_block = ko.gaussian_kernel(X, X[idx], 0.4)
    assert np.array_equal(col_block[idx], ko.gaussian_kernel(X[idx], X[idx], 0.4))


def test_node_constructors_reject_bad_arguments():
    import keystone_b200 as ks
    for g in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError):
            ks.GaussianKernelGenerator(g)
    gen = ks.GaussianKernelGenerator(1.0)
    with pytest.raises(ValueError):
        ks.KernelRidgeRegression(gen, 0.1, 0, 1)
    with pytest.raises(ValueError):
        ks.KernelRidgeRegression(gen, 0.1, 4, 0)
    with pytest.raises(ValueError):
        ks.KernelRidgeRegression(gen, -1.0, 4, 1)


def test_block_permuter_gives_one_permutation_per_epoch():
    import keystone_b200 as ks
    est = ks.KernelRidgeRegression(ks.GaussianKernelGenerator(1.0), 0.1, 64, 3, block_permuter=5)
    order = est.block_order(230)
    assert order.shape == (3, 4) and order.dtype == np.int32
    for row in order:
        assert sorted(row) == [0, 1, 2, 3]
    assert ks.KernelRidgeRegression(ks.GaussianKernelGenerator(1.0), 0.1, 64, 3).block_order(230) is None
