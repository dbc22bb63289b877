"""Sparse L-BFGS least squares (SparseLBFGSwithL2, K/nodes/learning/LBFGS.scala:208-281) as DESIGN.md section 20 defines it, on the
host: with an implicit ones column whose bias is regularised like every other unknown, the sparse fit is the no-intercept dense
algorithm (tests/lbfgs_oracle.py) on [A 1].  Reproduces the reference's sparse LBFGSSuite cases and checks the cost model."""
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lbfgs_oracle as lo  # noqa: E402

X_TRUE = np.array([[5.0, 4.0, 3.0, 2.0, -1.0], [3.0, -1.0, 2.0, -2.0, 1.0]])
DATA_MEAN = np.array([1.0, 0.0, 1.0, 2.0, 0.0])
EXTRA_BIAS = np.array([3.0, 4.0])


def sparse_suite_data(fit_intercept, seed=0):
    """LBFGSSuite.scala:62-108 with numpy data: a 128 x 5 Gaussian A and b = A x^T.  With an intercept the rows are A + dataMean
    (not centred) and the labels b + extraBias, so the expected bias is extraBias - x dataMean."""
    A = np.random.default_rng(seed).standard_normal((128, 5))
    B = A @ X_TRUE.T
    if not fit_intercept:
        return A, B
    return A + DATA_MEAN, B + EXTRA_BIAS


def sparse_fit(A, Y, fit_intercept, **kw):
    """The sparse algorithm through the dense oracle: (W, b or None, info)."""
    Aug = np.hstack([A, np.ones((A.shape[0], 1))]) if fit_intercept else A
    X, _, _, info = lo.fit(Aug, Y, fit_intercept=False, **kw)
    return (X[:-1], X[-1], info) if fit_intercept else (X, None, info)


@pytest.mark.parametrize("fit_intercept,tol", [(True, 1e-3), (False, 1e-4)])
def test_sparse_suite_cases(fit_intercept, tol):
    """The suite's own absolute tolerances at the default parameters (numCorrections 10, convergenceTol 1e-4, 100 iterations)."""
    A, B = sparse_suite_data(fit_intercept)
    W, b, info = sparse_fit(A, B, fit_intercept)
    pred = A @ W + (b if b is not None else 0.0)
    assert np.abs(pred - B).max() < tol
    assert np.abs(W - X_TRUE.T).max() < tol
    if fit_intercept:
        assert np.abs(b - (EXTRA_BIAS - X_TRUE @ DATA_MEAN)).max() < tol
    else:
        assert b is None
    assert info["iterations"] >= 1 and len(info["loss_history"]) == info["iterations"] + 1


def test_regularised_bias_is_the_zero_of_the_reference_gradient():
    """With lambda > 0 the fit converges to the zero of g = [A 1]^T ([A 1] x - Y) / N + lambda x (bias included, LBFGS.scala:117):
    the ridge solution on [A 1] with lambda N on every unknown."""
    A, B = sparse_suite_data(True, seed=3)
    lam = 0.05
    W, b, _ = sparse_fit(A, B, True, reg_param=lam, convergence_tol=1e-14, num_iterations=200)
    Aug = np.hstack([A, np.ones((A.shape[0], 1))])
    ref = np.linalg.solve(Aug.T @ Aug + lam * A.shape[0] * np.eye(6), Aug.T @ B)
    assert np.abs(np.vstack([W, b]) - ref).max() < 1e-9


def test_weight_and_cost_formulas():
    """weight = numIterations + 1 (LBFGS.scala:220) and CostModel.cost (:264-280)."""
    import keystone_b200 as ks
    est = ks.SparseLBFGSwithL2(ks.LeastSquaresSparseGradient(), num_iterations=37, sparse_overhead=5.0)
    assert est.weight == 38 and ks.SparseLBFGSwithL2().weight == 101
    n, d, k, s, m, cw, mw, nw = 10 ** 6, 10 ** 4, 3, 0.02, 4, 3.8e-4, 2.9e-1, 1.32
    flops = n * s * d * k / m
    scanned = n * d * s / m
    network = 2.0 * d * k * math.log(m) / math.log(2.0)
    ref = 37 * (5.0 * max(cw * flops, mw * scanned) + nw * network)
    assert est.cost(n, d, k, s, m, cw, mw, nw) == pytest.approx(ref, rel=1e-15)
    with pytest.raises(ValueError):
        ks.SparseLBFGSwithL2(ks.LeastSquaresDenseGradient())
    with pytest.raises(ValueError):
        ks.SparseLBFGSwithL2(num_iterations=0)
    with pytest.raises(ValueError):
        ks.SparseLBFGSwithL2(reg_param=float("nan"))


def test_cost_model_uses_the_sparse_node():
    """LeastSquaresEstimator's sparse row is SparseLBFGSwithL2(numIterations = 20).cost, and the suite's selections stand
    (LeastSquaresEstimatorSuite.scala:68-103)."""
    import keystone_b200 as ks
    est = ks.LeastSquaresEstimator(lam=0.1)
    for args in [(10 ** 6, 10000, 2, 0.01, 1), (10 ** 5, 300, 20, 0.3, 8)]:
        c = est.costs(*args)
        assert c["sparse_lbfgs"] == ks.SparseLBFGSwithL2(num_iterations=20).cost(*args, est.cpu_weight, est.mem_weight, est.network_weight)
    assert est.optimize(1_000_000, 1000, 1000) == "exact"
    assert est.optimize(1_000_000, 10000, 1000) == "block"
    assert est.optimize(1_000_000, 10000, 2, 0.01) == "sparse_lbfgs"
