"""fp64 NumPy restatement of the library's dense L-BFGS least squares (DenseLBFGSwithL2, K/nodes/learning/LBFGS.scala:135-192,
gradient K/nodes/learning/Gradient.scala:29-53; K/ = src/main/scala/keystoneml/ of the reference project), as DESIGN.md
section 14 defines it: exact centring, W_0 = 0, two-loop direction, exact step along it, the library's stop rules.
Host code, no GPU."""
import numpy as np


def fit(A, Y, fit_intercept=True, num_corrections=10, convergence_tol=1e-4, num_iterations=100, reg_param=0.0, shards=None,
        trace=None):
    """Returns (W, intercept or None, feature mean or None, info).  ``shards``: row-index arrays, one per rank; the gradient
    product and |A P|^2 are summed over them in rank order (what the all-reduce does), everything else is computed once.
    ``trace`` (a list) receives per step (f_old, g_old, P, alpha, f_new, g_new) for the line-search checks."""
    A = np.asarray(A, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    if Y.ndim == 1:
        Y = Y[:, None]
    n, d = A.shape
    k = Y.shape[1]
    lam, tol, m = float(reg_param), float(convergence_tol), int(num_corrections)
    if fit_intercept:
        mu, ybar = A.mean(0), Y.mean(0)
        Ac, Yc = A - mu, Y - ybar
    else:
        mu = ybar = None
        Ac, Yc = A, Y
    parts = [np.arange(n)] if shards is None else [np.asarray(s) for s in shards]

    def at(M):        # A_c^T M, summed over the shards
        return sum(Ac[s].T @ M[s] for s in parts)

    def sumsq(M):
        return sum(float((M[s] ** 2).sum()) for s in parts)

    W = np.zeros((d, k))
    R = Ac @ W - Yc
    g = at(R) / n + lam * W
    f = sumsq(R) / (2 * n) + lam / 2 * float((W ** 2).sum())
    losses, hist, iters, stop = [f], [], 0, "max_iterations"
    if np.abs(g).max() == 0.0:
        stop = "zero_gradient"
    for t in range(num_iterations if stop != "zero_gradient" else 0):
        q, a = g.copy(), []
        for s, y, rho in reversed(hist):
            ai = rho * float((s * q).sum())
            q -= ai * y
            a.append(ai)
        if hist:
            s, y, _ = hist[-1]
            q *= float((s * y).sum()) / float((y * y).sum())
        for (s, y, rho), ai in zip(hist, reversed(a)):
            q += (ai - rho * float((y * q).sum())) * s
        P = -q
        gP = float((g * P).sum())
        if gP >= 0.0:                       # not a descent direction after rounding: drop the history
            hist, P, gP = [], -g, -float((g * g).sum())
        Q = Ac @ P
        den = sumsq(Q) / n + lam * float((P * P).sum())
        if not den > 0.0:
            stop = "non_positive_curvature"
            break
        alpha = -gP / den                   # the exact minimiser along P
        W = W + alpha * P
        R = R + alpha * Q
        g_new = at(R) / n + lam * W
        f_new = sumsq(R) / (2 * n) + lam / 2 * float((W ** 2).sum())
        if trace is not None:
            trace.append((f, g, P, alpha, f_new, g_new))
        s, y = alpha * P, g_new - g
        g, f = g_new, f_new
        losses.append(f)
        iters = t + 1
        sy = float((s * y).sum())
        if not sy > 0.0:
            stop = "non_positive_curvature"
            break
        hist.append((s, y, 1.0 / sy))
        if len(hist) > m:
            hist.pop(0)
        gmax = float(np.abs(g).max())
        if gmax == 0.0:
            stop = "zero_gradient"
            break
        if t + 1 == num_iterations:
            stop = "max_iterations"
            break
        if tol > 0.0 and max(losses[-11:-1]) - f <= tol * abs(f):
            stop = "function_values_converged"
            break
        if tol > 0.0 and gmax <= max(tol * abs(f), 1e-8):
            stop = "gradient_converged"
            break
    return W, ybar, mu, {"loss_history": losses, "iterations": iters, "stop_reason": stop}


def apply(W, intercept, mean, A):
    """LinearMapper.apply (K/nodes/learning/LinearMapper.scala:35-46): (x - mean) W + intercept."""
    A = np.asarray(A, dtype=np.float64)
    out = (A - mean if mean is not None else A) @ W
    return out + intercept if intercept is not None else out


def ridge(A, Y, lam_n, fit_intercept=True):
    """The centred ridge solution (A_c^T A_c + lam_n I)^-1 A_c^T Y_c: LinearMapEstimator(lam_n), which the L-BFGS objective
    with reg_param = lam_n / N converges to."""
    A = np.asarray(A, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    if fit_intercept:
        A, Y = A - A.mean(0), Y - Y.mean(0)
    return np.linalg.solve(A.T @ A + lam_n * np.eye(A.shape[1]), A.T @ Y)


def suite_data(fit_intercept, seed=0):
    """LBFGSSuite's dense fixtures (T/nodes/learning/LBFGSSuite.scala:13-60): a 128 x 5 Gaussian matrix, the planted
    x = [[5, 4, 3, 2, -1], [3, -1, 2, -2, 1]]; with intercept the data is centred then shifted by dataMean = [1, 0, 1, 2, 0]
    and the labels get extraBias = [3, 4]."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((128, 5))
    x = np.array([[5.0, 4.0, 3.0, 2.0, -1.0], [3.0, -1.0, 2.0, -2.0, 1.0]])
    if not fit_intercept:
        return A, A @ x.T, x, None, None
    data_mean, extra_bias = np.array([1.0, 0.0, 1.0, 2.0, 0.0]), np.array([3.0, 4.0])
    A = A - A.mean(0) + data_mean
    return A, (A - data_mean) @ x.T + extra_bias, x, data_mean, extra_bias
