"""fp64 NumPy restatement of the library's logistic regression and multinomial naive Bayes (LogisticRegressionEstimator,
NaiveBayesEstimator; K/nodes/learning/{LogisticRegressionModel,NaiveBayesModel}.scala of the reference project, which wrap Spark
MLlib), as DESIGN.md section 22 defines them: the L-BFGS recursion and stop rules of tests/lbfgs_oracle.py with a strong-Wolfe line
search modelled on Breeze's, and MLlib's naive Bayes formulas.  Host code, no GPU.

``A`` may be a dense array or anything with ``@`` and ``.T`` (a scipy sparse matrix)."""
import math

import numpy as np

C1, C2 = 1e-4, 0.9
MAX_ZOOM, MAX_BRACKET = 10, 10
NUM_CORRECTIONS = 10


def _softmax_terms(Z, y):
    """Per row of the margins Z (n x (k-1), class 0 at margin 0): the data loss lse(0, z) - z_y, softmax(z) (columns 1..k-1) and
    onehot(y) (columns 1..k-1)."""
    m = np.maximum(0.0, Z.max(1)) if Z.shape[1] else np.zeros(Z.shape[0])
    E = np.exp(Z - m[:, None])
    s = np.exp(-m) + E.sum(1)
    onehot = np.zeros_like(Z)
    rows = np.nonzero(y > 0)[0]
    onehot[rows, y[rows] - 1] = 1.0
    loss = m + np.log(s) - (Z * onehot).sum(1)
    return loss, E / s[:, None], onehot


def loss_and_gradient(A, y, W, lam):
    """f(W) and g(W) of the logistic objective, directly from W."""
    n = A.shape[0]
    loss, P, onehot = _softmax_terms(np.asarray(A @ W), y)
    f = loss.sum() / n + lam / 2 * float((W * W).sum())
    g = np.asarray(A.T @ (P - onehot)) / n + lam * W
    return f, g


def _interp(l, r):
    """Breeze's safeguarded cubic between l = (t, f, dd) and r with l.t < r.t, clamped to [l + 0.1 w, l + 0.9 w]; the midpoint when
    the radical is negative or the result is not finite."""
    d1 = l[2] + r[2] - 3.0 * (l[1] - r[1]) / (l[0] - r[0])
    rad = d1 * d1 - l[2] * r[2]
    w = r[0] - l[0]
    if not rad >= 0.0:
        return l[0] + 0.5 * w
    d2 = math.sqrt(rad)
    with np.errstate(all="ignore"):
        t = r[0] - w * (r[2] + d2 - d1) / (r[2] - l[2] + 2.0 * d2)
    if not math.isfinite(t):
        return l[0] + 0.5 * w
    return min(max(t, l[0] + 0.1 * w), l[0] + 0.9 * w)


def line_search(phi, f0, dd0, t_init):
    """Strong-Wolfe search (DESIGN.md section 22).  phi(t) -> (f, dd).  Returns (alpha or None, evaluations)."""
    evals = [0]

    def ev(t):
        evals[0] += 1
        f, dd = phi(t)
        return (t, f, dd)

    def suff_fails(p, low):
        return not math.isfinite(p[1]) or p[1] > f0 + C1 * p[0] * dd0 or p[1] >= low[1]

    def zoom(low, hi):
        for _ in range(MAX_ZOOM):
            t = _interp(hi, low) if low[0] > hi[0] else _interp(low, hi)
            q = ev(t)
            if suff_fails(q, low):
                hi = q
            else:
                if abs(q[2]) <= C2 * abs(dd0):
                    return q[0]
                if q[2] * (hi[0] - low[0]) >= 0.0:
                    hi = low
                low = q
        return None

    if not dd0 < 0.0:
        return None, 0
    low, t = (0.0, f0, dd0), t_init
    for i in range(MAX_BRACKET):
        q = ev(t)
        if not math.isfinite(q[1]) or q[1] > f0 + C1 * t * dd0 or (q[1] >= low[1] and i > 0):
            return zoom(low, q), evals[0]
        if abs(q[2]) <= C2 * abs(dd0):
            return q[0], evals[0]
        if q[2] >= 0.0:
            return zoom(q, low), evals[0]
        low = q
        t *= 1.5
    return None, evals[0]


def _direction(g, hist):
    """The two-loop recursion of tests/lbfgs_oracle.py over hist = [(s, y, rho)], oldest first: -H g."""
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
    return -q


def logistic_fit(A, y, num_classes, reg_param=0.0, num_iters=100, convergence_tol=1e-4, trace=None):
    """Returns (W (d x (k-1)), info).  ``trace`` (a list) receives per accepted step (f0, dd0, alpha, f(alpha), phi'(alpha))."""
    y = np.asarray(y, dtype=np.int64)
    n, d = A.shape
    kk = int(num_classes) - 1
    lam, tol = float(reg_param), float(convergence_tol)
    W = np.zeros((d, kk))
    Z = np.zeros((n, kk))

    def at_point(Z, W):
        loss, P, onehot = _softmax_terms(Z, y)
        return loss.sum() / n + lam / 2 * float((W * W).sum()), np.asarray(A.T @ (P - onehot)) / n + lam * W

    f, g = at_point(Z, W)
    losses, hist, evals, iters, stop = [f], [], [], 0, "max_iterations"
    if np.abs(g).max() == 0.0:
        stop = "zero_gradient"
    failed_once, t = False, 0
    while t < num_iters and stop != "zero_gradient":
        P = _direction(g, hist)
        gP = float((g * P).sum())
        if gP >= 0.0:
            hist, P, gP = [], -g, -float((g * g).sum())
        Q = np.asarray(A @ P)
        WW, WP, PP = float((W * W).sum()), float((W * P).sum()), float((P * P).sum())

        def phi(s):
            with np.errstate(over="ignore", invalid="ignore"):
                loss, Pr, onehot = _softmax_terms(Z + s * Q, y)
                return (loss.sum() / n + 0.5 * lam * (WW + 2.0 * s * WP + s * s * PP),
                        float(((Pr - onehot) * Q).sum()) / n + lam * (WP + s * PP))

        alpha, ne = line_search(phi, f, gP, 1.0 / math.sqrt(PP) if t == 0 and PP > 0 else 1.0)
        evals.append(ne)
        if alpha is not None and alpha * math.sqrt(float((g * g).sum())) < 1e-10:
            alpha = None
        if alpha is None:
            if failed_once:
                stop = "line_search_failed"
                break
            failed_once, hist = True, []
            continue
        if trace is not None:
            trace.append((f, gP, alpha) + phi(alpha))
        W = W + alpha * P
        Z = Z + alpha * Q
        f_new, g_new = at_point(Z, W)
        s_, y_ = alpha * P, g_new - g
        g, f = g_new, f_new
        losses.append(f)
        iters = t + 1
        sy = float((s_ * y_).sum())
        if not sy > 0.0:
            stop = "non_positive_curvature"
            break
        hist.append((s_, y_, 1.0 / sy))
        if len(hist) > NUM_CORRECTIONS:
            hist.pop(0)
        gmax = float(np.abs(g).max())
        if gmax == 0.0:
            stop = "zero_gradient"
            break
        if t + 1 == num_iters:
            stop = "max_iterations"
            break
        if tol > 0.0 and max(losses[-11:-1]) - f <= tol * abs(f):
            stop = "function_values_converged"
            break
        if tol > 0.0 and gmax <= max(tol * abs(f), 1e-8):
            stop = "gradient_converged"
            break
        t += 1
    return W, {"loss_history": losses, "iterations": iters, "stop_reason": stop, "line_search_evals": evals}


def logistic_predict(W, A):
    """MLlib's predict: the first maximum of [0, A W] (float class ids)."""
    Z = np.asarray(A @ W)
    return np.argmax(np.hstack([np.zeros((Z.shape[0], 1)), Z]), axis=1).astype(np.float64)


def naive_bayes_fit(A, y, num_classes, lam=1.0):
    """(pi (k), theta (k x d)) of MLlib's multinomial NaiveBayes.train."""
    y = np.asarray(y, dtype=np.int64)
    k = int(num_classes)
    d = A.shape[1]
    Y = np.zeros((A.shape[0], k))
    Y[np.arange(A.shape[0]), y] = 1.0
    S = np.asarray(A.T @ Y).T      # k x d
    counts = Y.sum(0)
    pi = np.log(counts + lam) - math.log(counts.sum() + k * lam)
    theta = np.log(S + lam) - np.log(S.sum(1) + d * lam)[:, None]
    return pi, theta
