"""The fp64 oracle of logistic regression and naive Bayes (tests/classifier_oracle.py) against the reference's own suites
(LogisticRegressionModelSuite, NaiveBayesModelSuite; T/ = src/test/scala/keystoneml/ of the reference project), the strong-Wolfe
conditions, scipy's L-BFGS-B on the same objective and a direct per-class naive Bayes formula.  CPU only."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import classifier_oracle as co  # noqa: E402


class JavaRandom:
    """java.util.Random (the JDK's documented LCG, nextDouble and the polar nextGaussian); scala.util.Random(seed) wraps it."""

    MASK = (1 << 48) - 1

    def __init__(self, seed: int):
        self.seed = (seed ^ 0x5DEECE66D) & self.MASK
        self.next_gaussian = None

    def _next(self, bits: int) -> int:
        self.seed = (self.seed * 0x5DEECE66D + 0xB) & self.MASK
        return self.seed >> (48 - bits)

    def nextDouble(self) -> float:
        return ((self._next(26) << 27) + self._next(27)) * 2.0 ** -53

    def nextGaussian(self) -> float:
        if self.next_gaussian is not None:
            g, self.next_gaussian = self.next_gaussian, None
            return g
        while True:
            v1, v2 = 2 * self.nextDouble() - 1, 2 * self.nextDouble() - 1
            s = v1 * v1 + v2 * v2
            if 0 < s < 1:
                break
        mul = math.sqrt(-2 * math.log(s) / s)
        self.next_gaussian = v2 * mul
        return v1 * mul


def logistic_input(offset, scale, n, seed):
    """LogisticRegressionModelSuite.generateLogisticInput: (labels, n x 1 features)."""
    rnd = JavaRandom(seed)
    x = np.array([rnd.nextGaussian() for _ in range(n)])
    y = np.array([1 if rnd.nextDouble() < 1.0 / (1.0 + math.exp(-(offset + scale * v))) else 0 for v in x])
    return y, x[:, None]


MULTI_WEIGHTS = [-0.57997, 0.912083, -0.371077, -0.819866, 2.688191, -0.16624, -0.84355, -0.048509, -0.301789, 4.170682]
MULTI_WEIGHTS_R = np.array([-0.5837166, 0.9285260, -0.3783612, -0.8123411, 2.6228269, -0.1691865, -0.811048, -0.0646380])


def multinomial_input(n, seed, weights=MULTI_WEIGHTS, d=4):
    """LogisticRegressionModelSuite.generateMultinomialLogisticInput with addIntercept = false: (labels, n x 4 features).  The
    suite's weights vector has 10 entries, so with xDim = 4 it yields nClasses = 10 / 4 + 1 = 3 and reads weights[i * 4 + j].  The
    suite's scaling by xVariance and xMean writes into ``vector.toArray``, which for a Breeze DenseVector is a copy: the features
    stay standard normal, and the labels are drawn from those unscaled features."""
    rnd = JavaRandom(seed)
    X = np.array([[rnd.nextGaussian() for _ in range(d)] for _ in range(n)])
    k = len(weights) // d + 1
    y = np.zeros(n, dtype=np.int64)
    for i in range(n):
        margins = [0.0] + [sum(weights[c * d + j] * X[i, j] for j in range(d)) for c in range(k - 1)]
        mx = max(margins)
        if mx > 0:
            margins = [m - mx for m in margins]
        probs = [math.exp(m) for m in margins]
        norm = sum(probs)
        probs = [p / norm for p in probs]
        for c in range(1, k):
            probs[c] += probs[c - 1]
        p = rnd.nextDouble()
        y[i] = next((c for c in range(k) if p < probs[c]), 0)
    return y, X


NB_PI = np.array([0.5, 0.1, 0.4])
NB_THETA = np.array([[0.7, 0.1, 0.1, 0.1], [0.1, 0.7, 0.1, 0.1], [0.1, 0.1, 0.7, 0.1]])


def naive_bayes_input(n, seed, samples=10):
    """NaiveBayesModelSuite.generateNaiveBayesInput (multinomial) with numpy draws from the same distributions."""
    rng = np.random.default_rng(seed)
    y = rng.choice(len(NB_PI), n, p=NB_PI)
    X = np.stack([rng.multinomial(samples, NB_THETA[c]) for c in y]).astype(np.float64)
    return y, X


# ------------------------------------------------------------------------------------------------ the JDK generator
def test_java_random_matches_the_jdk():
    """Values of new java.util.Random(42): nextInt() is next(32) as a signed int; the first nextDouble and nextGaussian."""
    r = JavaRandom(42)
    v = r._next(32)
    assert (v - (1 << 32) if v >= 1 << 31 else v) == -1170105035
    assert JavaRandom(42).nextDouble() == pytest.approx(0.7275636800328681, abs=0)
    assert JavaRandom(42).nextGaussian() == pytest.approx(1.1419053154730547, rel=1e-15)


# ------------------------------------------------------------------------------------------------ the reference suites
def test_binary_suite():
    """'logistic regression with LBFGS': weight within 0.03 of -0.8 and validation accuracy > 0.65 at the defaults."""
    y, X = logistic_input(0.0, -0.8, 10000, 42)
    W, info = co.logistic_fit(X, y, 2)
    assert abs(W[0, 0] - (-0.8)) <= 0.03
    yv, Xv = logistic_input(0.0, -0.8, 10000, 17)
    assert (co.logistic_predict(W, Xv) == yv).mean() > 0.65
    assert info["iterations"] >= 1 and len(info["loss_history"]) == info["iterations"] + 1


def test_multinomial_suite():
    """'multinomial logistic regression with LBFGS': weights within 0.05 of the suite's R values, validation accuracy > 0.47."""
    y, X = multinomial_input(10000, 42)
    W, info = co.logistic_fit(X, y, 3, num_iters=200, convergence_tol=1e-15)
    weights = W.T.ravel()                      # MLlib's class-major layout
    assert np.abs(weights - MULTI_WEIGHTS_R).max() <= 0.05, (weights, info["stop_reason"])
    yv, Xv = multinomial_input(10000, 17)
    assert (co.logistic_predict(W, Xv) == yv).mean() > 0.47


def test_naive_bayes_suite():
    """'Naive Bayes Multinomial': exp(pi) and exp(theta) within 0.05, and >= 80 % of the validation predictions right."""
    y, X = naive_bayes_input(1000, 42)
    pi, theta = co.naive_bayes_fit(X, y, 3, 1.0)
    assert np.abs(np.exp(pi) - NB_PI).max() <= 0.05
    assert np.abs(np.exp(theta) - NB_THETA).max() <= 0.05
    yv, Xv = naive_bayes_input(1000, 17)
    assert (np.argmax(Xv @ theta.T + pi, axis=1) == yv).mean() >= 0.8


# ------------------------------------------------------------------------------------------------ the line search
@pytest.mark.parametrize("k,lam", [(2, 0.0), (3, 1e-3), (5, 0.1)])
def test_steps_are_strong_wolfe_and_monotone(k, lam):
    rng = np.random.default_rng(k)
    X = rng.standard_normal((400, 7)) * 2.0
    y = rng.integers(0, k, 400)
    trace = []
    _, info = co.logistic_fit(X, y, k, reg_param=lam, num_iters=30, convergence_tol=0.0, trace=trace)
    assert len(trace) == info["iterations"] >= 5
    for f0, dd0, alpha, fa, dda in trace:
        assert fa <= f0 + co.C1 * alpha * dd0
        assert abs(dda) <= co.C2 * abs(dd0)
    assert all(b <= a for a, b in zip(info["loss_history"], info["loss_history"][1:]))
    assert info["loss_history"][0] == pytest.approx(math.log(k), rel=1e-15)


def test_loss_and_gradient_against_finite_differences():
    rng = np.random.default_rng(3)
    X = rng.standard_normal((50, 4))
    y = rng.integers(0, 4, 50)
    W = rng.standard_normal((4, 3)) * 0.3
    f, g = co.loss_and_gradient(X, y, W, 0.2)
    E = rng.standard_normal(W.shape)
    h = 1e-6
    fd = (co.loss_and_gradient(X, y, W + h * E, 0.2)[0] - co.loss_and_gradient(X, y, W - h * E, 0.2)[0]) / (2 * h)
    assert fd == pytest.approx(float((g * E).sum()), rel=1e-7)


@pytest.mark.parametrize("k,lam", [(2, 1e-2), (4, 0.1)])
def test_converged_weights_match_scipy(k, lam):
    """At lambda > 0 the converged oracle W is scipy's L-BFGS-B minimiser of the same objective (an independent check of f and g)."""
    scipy_opt = pytest.importorskip("scipy.optimize")
    rng = np.random.default_rng(11 + k)
    X = rng.standard_normal((600, 6))
    y = rng.integers(0, k, 600)
    W, info = co.logistic_fit(X, y, k, reg_param=lam, num_iters=500, convergence_tol=1e-12)

    def fg(w):
        f, g = co.loss_and_gradient(X, y, w.reshape(6, k - 1), lam)
        return f, g.ravel()

    res = scipy_opt.minimize(fg, np.zeros(6 * (k - 1)), jac=True, method="L-BFGS-B",
                             options={"maxiter": 10000, "ftol": 1e-16, "gtol": 1e-13})
    Ws = res.x.reshape(6, k - 1)
    assert np.linalg.norm(W - Ws) / np.linalg.norm(Ws) <= 1e-6, info["stop_reason"]


def test_separable_data_stays_finite():
    X = np.concatenate([np.linspace(0.5, 3, 50), -np.linspace(0.5, 3, 50)])[:, None]
    y = np.array([1] * 50 + [0] * 50)
    W, info = co.logistic_fit(X, y, 2, num_iters=100, convergence_tol=0.0)
    assert np.isfinite(W).all() and np.isfinite(info["loss_history"]).all()
    assert W[0, 0] > 0


def test_naive_bayes_matches_per_class_formula():
    rng = np.random.default_rng(5)
    X = rng.random((300, 9)) * 3.0
    y = rng.integers(0, 4, 300)
    pi, theta = co.naive_bayes_fit(X, y, 4, 0.7)
    for c in range(4):
        rows = X[y == c]
        assert pi[c] == pytest.approx(math.log(len(rows) + 0.7) - math.log(300 + 4 * 0.7), rel=1e-14)
        tot = rows.sum()
        for j in range(9):
            assert theta[c, j] == pytest.approx(math.log(rows[:, j].sum() + 0.7) - math.log(tot + 9 * 0.7), rel=1e-12, abs=1e-14)
