"""Dense L-BFGS least squares on the host: the fp64 oracle (tests/lbfgs_oracle.py) against LBFGSSuite's dense known answers and
the closed-form ridge solution, the line-search and stopping properties the device fit shares with it, the two-rank algebra,
and the node's weight, cost and argument checks.  No GPU needed."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lbfgs_oracle as lo  # noqa: E402


@pytest.mark.parametrize("fit_intercept", [True, False])
def test_suite_known_answers(fit_intercept):
    """T/nodes/learning/LBFGSSuite.scala:13-60 at the default parameters (numCorrections 10, convergenceTol 1e-4,
    numIterations 100, regParam 0); the reference asserts 1e-5, the fp64 oracle meets 1e-8."""
    A, B, x, data_mean, extra_bias = lo.suite_data(fit_intercept)
    W, b, mu, info = lo.fit(A, B, fit_intercept=fit_intercept)
    assert np.abs(lo.apply(W, b, mu, A) - B).max() < 1e-8
    assert np.abs(W - x.T).max() < 1e-8
    if fit_intercept:
        assert np.abs(b - extra_bias).max() < 1e-8
        assert np.abs(mu - data_mean).max() < 1e-8
    else:
        assert b is None and mu is None
    assert info["stop_reason"] in ("gradient_converged", "function_values_converged", "zero_gradient")
    assert info["iterations"] <= 100


@pytest.mark.parametrize("lam", [0.0, 1e-3, 0.5])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_converged_fit_is_the_centred_ridge_solution(lam, fit_intercept):
    """min |A_c W - Y_c|^2 / (2N) + lam/2 |W|^2 is LinearMapEstimator(N lam)."""
    rng = np.random.default_rng(3)
    n, d, k = 300, 40, 3
    A = rng.standard_normal((n, d)) @ np.diag(np.linspace(0.3, 3.0, d)) + 2.0
    Y = A @ rng.standard_normal((d, k)) + 0.3 * rng.standard_normal((n, k)) - 1.0
    W, _, _, info = lo.fit(A, Y, fit_intercept=fit_intercept, convergence_tol=1e-14, num_iterations=500, reg_param=lam)
    ref = lo.ridge(A, Y, n * lam, fit_intercept)
    assert np.linalg.norm(W - ref) / np.linalg.norm(ref) < 1e-8, info


def test_every_step_satisfies_strong_wolfe_and_the_loss_never_increases():
    rng = np.random.default_rng(5)
    n, d, k = 200, 30, 2
    A = rng.standard_normal((n, d)) @ np.diag(np.linspace(0.1, 1.0, d))
    Y = rng.standard_normal((n, k))
    trace = []
    _, _, _, info = lo.fit(A, Y, num_corrections=4, convergence_tol=0.0, num_iterations=25, reg_param=0.01, trace=trace)
    assert len(trace) == info["iterations"] == 25
    c1, c2 = 0.49, 1e-6   # the exact step meets any c1 <= 1/2 (f_new = f + alpha g.P / 2) and any c2 (g_new.P = 0)
    for f, g, P, alpha, f_new, g_new in trace:
        gP = float((g * P).sum())
        assert gP < 0 and alpha > 0
        if f - f_new > 1e-12 * abs(f):
            assert f_new <= f + c1 * alpha * gP
        assert abs(float((g_new * P).sum())) <= c2 * abs(gP) + 1e-15
    losses = info["loss_history"]
    assert all(b <= a * (1 + 1e-15) for a, b in zip(losses, losses[1:]))


@pytest.mark.parametrize("iters", [1, 3, 8])
def test_zero_tolerance_runs_exactly_num_iterations(iters):
    rng = np.random.default_rng(iters)
    A = rng.standard_normal((100, 20))
    Y = rng.standard_normal((100, 2))
    _, _, _, info = lo.fit(A, Y, convergence_tol=0.0, num_iterations=iters)
    assert info["iterations"] == iters and info["stop_reason"] == "max_iterations"
    assert len(info["loss_history"]) == iters + 1


def test_stop_rules():
    rng = np.random.default_rng(1)
    A = rng.standard_normal((100, 10))
    Y = A @ rng.standard_normal((10, 1)) + 0.1 * rng.standard_normal((100, 1))
    _, _, _, info = lo.fit(A, Y, convergence_tol=1e-3, num_iterations=100)
    assert info["stop_reason"] in ("function_values_converged", "gradient_converged")
    assert info["iterations"] < 100
    _, _, _, info = lo.fit(A, np.zeros((100, 1)), convergence_tol=0.0, num_iterations=5)
    assert info["stop_reason"] == "zero_gradient" and info["iterations"] == 0


@pytest.mark.parametrize("fit_intercept", [True, False])
def test_two_rank_algebra_equals_one_rank(fit_intercept):
    """The device sums the gradient product and |A_c P|^2 over the ranks' row shards, then runs the identical recursion on
    every rank: uneven shards give the one-rank fit (up to the order of the shard sums, which 12 steps amplify)."""
    rng = np.random.default_rng(9)
    n, d, k = 257, 33, 4
    A = rng.standard_normal((n, d)) + 0.5
    Y = rng.standard_normal((n, k))
    one = lo.fit(A, Y, fit_intercept=fit_intercept, convergence_tol=0.0, num_iterations=12, reg_param=0.02)
    two = lo.fit(A, Y, fit_intercept=fit_intercept, convergence_tol=0.0, num_iterations=12, reg_param=0.02,
                 shards=[np.arange(0, 100), np.arange(100, n)])
    assert np.linalg.norm(one[0] - two[0]) / np.linalg.norm(one[0]) < 1e-6
    assert np.allclose(one[3]["loss_history"], two[3]["loss_history"], rtol=1e-10, atol=0)


def test_weight_and_cost_match_the_reference_formulas():
    import keystone_b200 as ks
    e = ks.DenseLBFGSwithL2(ks.LeastSquaresDenseGradient(), num_iterations=37)
    assert e.weight == 38                                              # LBFGS.scala:144
    n, d, k, m, cw, mw, nw = 1_000_000, 16384, 147, 4, 3.8e-4, 2.9e-1, 1.32
    flops = n * d * k / m                                              # LBFGS.scala:185-190
    scanned = n * d / m
    network = 2.0 * d * k * math.log(m) / math.log(2.0)
    assert e.cost(n, d, k, 1.0, m, cw, mw, nw) == pytest.approx(37 * (max(cw * flops, mw * scanned) + nw * network), rel=1e-15)
    # LeastSquaresEstimator.default is DenseLBFGSwithL2 with 20 iterations (LeastSquaresEstimator.scala:55-57)
    est = ks.LeastSquaresEstimator(num_machines=m)
    assert est.costs(n, d, k, 1.0, m)["dense_lbfgs"] == ks.DenseLBFGSwithL2(num_iterations=20).cost(n, d, k, 1.0, m, cw, mw, nw)
    defaults = ks.DenseLBFGSwithL2()
    assert (defaults.fit_intercept, defaults.num_corrections, defaults.convergence_tol, defaults.num_iterations,
            defaults.reg_param) == (True, 10, 1e-4, 100, 0.0)
    assert isinstance(defaults.gradient, ks.LeastSquaresDenseGradient)


@pytest.mark.parametrize("kwargs", [dict(num_corrections=0), dict(num_iterations=0), dict(reg_param=-1.0),
                                    dict(reg_param=float("nan")), dict(reg_param=float("inf")), dict(convergence_tol=-1e-4),
                                    dict(convergence_tol=float("nan")), dict(precision="bf16"), dict(gradient=object())])
def test_node_argument_checks(kwargs):
    import keystone_b200 as ks
    with pytest.raises(ValueError):
        ks.DenseLBFGSwithL2(**kwargs)
