"""fp64 NumPy oracle of the mixture and k-means fits (K/nodes/learning/{GaussianMixtureModelEstimator,KMeansPlusPlus}.scala), with the
uniforms injected and the draw rule of include/keystone_b200.h (DESIGN.md section 17).

X is N x dim (one sample per row).  Means and variances are returned dim x K like the reference's GaussianMixtureModel.  The E-step
log-likelihoods use the reference's expanded Mahalanobis form, as fv_oracle.gmm_posteriors does; k-means distances use the direct
form 1/2 |x - c|^2, the quantity the reference's expanded form approximates."""
import math

import numpy as np

SUM_ROWS = 256


def _tree_block_sums(d: np.ndarray) -> np.ndarray:
    """B_b: the tree sum of rows [256 b, 256 b + 256) of d (zeros past the end), pairs at distance 128, 64, ..., 1."""
    nb = (d.size + SUM_ROWS - 1) // SUM_ROWS
    v = np.zeros(nb * SUM_ROWS)
    v[:d.size] = d
    v = v.reshape(nb, SUM_ROWS)
    h = SUM_ROWS // 2
    while h > 0:
        v = v[:, :h] + v[:, h:2 * h]
        h //= 2
    return v[:, 0]


def _half_sq_dist(X: np.ndarray, c: np.ndarray) -> np.ndarray:
    """1/2 sum_d (x_d - c_d)^2, the sum over d in order (no fused multiply-add, as the device kernel)."""
    acc = np.zeros(X.shape[0])
    for j in range(X.shape[1]):
        t = X[:, j] - c[j]
        acc = acc + t * t
    return 0.5 * acc


def draw_row(d: np.ndarray, u: float) -> int:
    """The row the k-means++ rule picks for uniform u given the weights d (include/keystone_b200.h)."""
    B = _tree_block_sums(d)
    W = 0.0
    for b in B:
        W = W + b
    if not W > 0.0:
        raise ValueError("fewer distinct points than centres")
    target = u * W
    base, pick, pbase, last, lbase = 0.0, -1, 0.0, -1, 0.0
    for b, bs in enumerate(B):
        nxt = base + bs
        if bs > 0.0:
            last, lbase = b, base
        if nxt > target:
            pick, pbase = b, base
            break
        base = nxt
    if pick < 0:
        pick, pbase = last, lbase
    r0, r1 = pick * SUM_ROWS, min(d.size, (pick + 1) * SUM_ROWS)
    s, last_pos = 0.0, r0
    for r in range(r0, r1):
        s = s + d[r]
        if d[r] > 0.0:
            last_pos = r
        if pbase + s > target:
            return r
    return last_pos


def kmeans_pp_seeds(X: np.ndarray, u) -> list:
    """k-means++ seeding (KMeansPlusPlus.scala:100-124) with one uniform per centre."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    seeds = [min(int(math.floor(u[0] * n)), n - 1)]
    d = None
    for j in range(1, len(u)):
        nd = _half_sq_dist(X, X[seeds[-1]])
        d = nd if d is None else np.minimum(nd, d)
        seeds.append(draw_row(d, u[j]))
    return seeds


def assign(X: np.ndarray, means: np.ndarray):
    """KMeansModel.apply: (first nearest centre index per row, its 1/2 |x - c|^2); means K x dim."""
    dist = np.stack([_half_sq_dist(X, m) for m in np.atleast_2d(means)], 1)
    idx = np.argmin(dist, 1)
    return idx, dist[np.arange(X.shape[0]), idx]


def kmeans_fit(X, k: int, max_iterations: int, stop_tolerance: float, u):
    """KMeansPlusPlusEstimator.fit: returns dict(means K x dim, seeds, iterations, costs, assignment of the last pass)."""
    X = np.asarray(X, dtype=np.float64)
    seeds = kmeans_pp_seeds(X, u[:k])
    means = X[seeds].copy()
    costs, it = [], 0
    while it < max_iterations:
        idx, best = assign(X, means)
        costs.append(best.mean())
        mass = np.bincount(idx, minlength=k).astype(np.float64)
        if (mass == 0).any():
            raise ValueError(f"cluster {int(np.argmin(mass))} is empty")
        A = np.zeros((X.shape[0], k))
        A[np.arange(X.shape[0]), idx] = 1.0
        means = (A.T @ X) / mass[:, None]
        it += 1
        if it > 1 and not ((costs[-2] - costs[-1]) >= stop_tolerance * abs(costs[-2])):
            break
    return {"means": means, "seeds": seeds, "iterations": it, "costs": costs, "assignment": idx}


def xerox_lse(llh: np.ndarray) -> np.ndarray:
    """The reference's incremental log-sum-exp over components 1..K-1 in order (GaussianMixtureModelEstimator.scala:127-146)."""
    lse = llh[:, 0].copy()
    for c in range(1, llh.shape[1]):
        l = llh[:, c]
        delta = lse - l
        inc = np.where(delta > 30.0, delta, np.where(delta > -30.0, np.log(np.exp(np.clip(delta, -30.0, 30.0)) + 1.0), 0.0))
        lse = inc + l
    return lse


def log_likelihoods(X, means_kd, vars_kd, weights):
    D = X.shape[1]
    sq = (X * X) @ (0.5 / vars_kd).T - X @ (means_kd / vars_kd).T + 0.5 * (means_kd * means_kd / vars_kd).sum(1)[None, :]
    return (-0.5 * D * math.log(2 * math.pi) - 0.5 * np.log(vars_kd).sum(1) + np.log(weights))[None, :] - sq


def gmm_fit(X, k: int, max_iterations: int = 100, min_cluster_size: float = 40, stop_tolerance: float = 1e-4,
            weight_threshold: float = 1e-4, small_variance_threshold: float = 1e-2, absolute_variance_threshold: float = 1e-9,
            init: str = "kmeans++", uniforms=None):
    """GaussianMixtureModelEstimator.fit.  uniforms: k values (k-means++) or k x dim (random).  Returns dict(means, variances (dim x K),
    weights, weight_threshold (1e-4, the reference model's default), iterations, stop_reason, costs, seeds)."""
    X = np.asarray(X, dtype=np.float64)
    n, D = X.shape
    XSq = X * X
    mean_g = X.sum(0) / n
    var_g = XSq.sum(0) / n - mean_g * mean_g
    lb = np.maximum(small_variance_threshold * var_g, absolute_variance_threshold)
    seeds = None
    if init == "kmeans++":
        km = kmeans_fit(X, k, 1, 1e-3, np.asarray(uniforms))
        seeds = km["seeds"]
        idx, _ = assign(X, km["means"])
        A = np.zeros((n, k))
        A[np.arange(n), idx] = 1.0
        mass = A.sum(0)
        if (mass == 0).any():
            raise ValueError(f"cluster {int(np.argmin(mass))} is empty")
        w = mass / n
        inv = 1.0 / mass
        mu = inv[:, None] * (A.T @ X)
        var = inv[:, None] * (A.T @ XSq) - mu * mu
    else:
        U = np.asarray(uniforms, dtype=np.float64).reshape(k, D)
        lo, hi = X.min(0), X.max(0)
        rng = hi - lo
        mu = U * rng[None, :] + lo[None, :]
        var = np.tile(0.1 * (rng * rng), (k, 1))
        w = np.full(k, 1.0 / k)
    var = np.maximum(var, lb[None, :])
    costs, it, reason = [], 0, "max_iterations"
    while it < max_iterations:
        llh = log_likelihoods(X, mu, var, w)
        costs.append(xerox_lse(llh).mean())
        it += 1
        if it > 1 and not ((costs[-1] - costs[-2]) >= stop_tolerance * abs(costs[-2])):
            reason = "cost"
            break
        q = np.exp(llh - llh.max(1, keepdims=True))
        q /= q.sum(1, keepdims=True)
        q = np.where(q > weight_threshold, q, 0.0)
        q /= q.sum(1, keepdims=True)
        qs = q.sum(0)
        if (qs < min_cluster_size).any():
            reason = "min_cluster_size"
            break
        w = qs / n
        inv = 1.0 / qs
        mu = inv[:, None] * (q.T @ X)
        var = np.maximum(inv[:, None] * (q.T @ XSq) - mu * mu, lb[None, :])
    return {"means": mu.T.copy(), "variances": var.T.copy(), "weights": w, "weight_threshold": 1e-4, "iterations": it,
            "stop_reason": reason, "costs": costs, "seeds": seeds}


def default_uniforms(k: int, dim: int = 0, seed: int = 0, init: str = "kmeans++") -> np.ndarray:
    """The uniforms the Python nodes draw: numpy.random.default_rng(seed).random(k) or .random((k, dim))."""
    rng = np.random.default_rng(seed)
    return rng.random(k) if init == "kmeans++" else rng.random((k, dim))


def mixture_sample(n: int, D: int, K: int, seed: int = 0, spread: float = 6.0):
    """A seeded synthetic mixture: K well-separated Gaussian clusters with per-dimension scales, rounded to fp32."""
    rng = np.random.default_rng(seed)
    centres = rng.normal(0.0, spread, (K, D))
    scales = rng.uniform(0.5, 1.5, (K, D))
    lab = rng.integers(0, K, n)
    X = centres[lab] + scales[lab] * rng.normal(0.0, 1.0, (n, D))
    return X.astype(np.float32).astype(np.float64)
