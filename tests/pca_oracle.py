"""fp64 NumPy oracle of the covariance-based transforms (K/nodes/learning/{PCA,DistributedPCA,ApproximatePCA,ZCAWhitener}.scala).

The reference computes in fp32 LAPACK (sgesvd) and draws its sketch matrix from Breeze's MersenneTwister; this oracle restates the
same algorithms in fp64 with the test matrix passed in, so the device can be compared on the same arrays."""
import math

import numpy as np


def sign_convention(pca: np.ndarray) -> np.ndarray:
    """PCAEstimator.enforceMatlabPCASignConvention (PCA.scala:238-247): a column is flipped unless its maximum element equals its
    maximum absolute value (ties keep +)."""
    pca = np.asarray(pca, dtype=np.float64)
    signs = np.where(pca.max(0) == np.abs(pca).max(0), 1.0, -1.0)
    return pca * signs


def compute_pca(X: np.ndarray, dims: int) -> np.ndarray:
    """PCAEstimator.computePCA (PCA.scala:171-199): right singular vectors of the centred data, sign convention, first dims."""
    Xc = X - X.mean(0)
    _, _, vt = np.linalg.svd(Xc, full_matrices=Xc.shape[0] < Xc.shape[1])  # all d right singular vectors, never an N x N U
    return sign_convention(vt.T)[:, :dims]


def singular_values_sq(X: np.ndarray) -> np.ndarray:
    """Eigenvalues of X_c^T X_c in descending order (the squared singular values of the centred data)."""
    s = np.linalg.svd(X - X.mean(0), compute_uv=False)
    return s ** 2


def compute_pca_eigh(X: np.ndarray, dims: int):
    """The device's route: eigenpairs of the centred covariance, descending, sign convention, first dims."""
    Xc = X - X.mean(0)
    lam, V = np.linalg.eigh(Xc.T @ Xc)
    return sign_convention(V[:, ::-1])[:, :dims], lam[::-1]


def tsqr_r(shards):
    """TSQR's R: QR of every shard, then QR of the stacked R factors."""
    rs = [np.linalg.qr(s, mode="r") for s in shards if s.shape[0] > 0]
    return np.linalg.qr(np.concatenate(rs, 0), mode="r")


def distributed_pca(shards, dims: int) -> np.ndarray:
    """DistributedPCAEstimator.computePCA (DistributedPCA.scala:34-56): global mean, TSQR of the centred shards, SVD of R."""
    n = sum(s.shape[0] for s in shards)
    mean = sum(s.sum(0) for s in shards) / n
    R = tsqr_r([s - mean for s in shards])
    _, _, vt = np.linalg.svd(R)
    return sign_convention(vt.T)[:, :dims]


def householder_q(Y: np.ndarray) -> np.ndarray:
    """QRUtils.qrQR(Y)._1: the thin Householder Q."""
    return np.linalg.qr(Y, mode="reduced")[0]


def cholqr_pass(Y: np.ndarray, shift: bool, shards=None, used=None) -> np.ndarray:
    """One CholeskyQR pass as the device runs it: G = sum over shards of Y_s^T Y_s, L L^T = G (+ sigma I), Y L^-T.  A plain pass
    whose factor shows max L_ii / min L_ii > 1e5 (or fails) is repeated with the shift."""
    n, l = Y.shape
    G = Y.T @ Y if shards is None else sum(Y[a:b].T @ Y[a:b] for a, b in shards)
    sigma = 11.0 * (n * l + l * (l + 1)) * 2.0 ** -53 * np.trace(G)
    for use_shift in ([True] if shift else [False, True]):
        try:
            L = np.linalg.cholesky(G + (sigma * np.eye(l) if use_shift else 0.0))
        except np.linalg.LinAlgError:
            continue
        dg = np.abs(np.diag(L))
        if use_shift or (dg.min() > 0 and dg.max() / dg.min() <= 1e5):
            break
    if used is not None:
        used.append(use_shift)
    return np.linalg.solve(L, Y.T).T


def shifted_cholqr3(Y: np.ndarray, shards=None) -> np.ndarray:
    """Shifted CholeskyQR3: a shifted pass, then plain ones.  When a later pass needs the shift too (an exactly rank-deficient Y),
    passes continue until one from the third on runs plain (at most 8)."""
    used = []
    Q = Y
    for i in range(8):
        Q = cholqr_pass(Q, i == 0, shards, used)
        if i >= 2 and not used[-1]:
            break
    return Q


def approximate_q(A: np.ndarray, omega: np.ndarray, q: int, qr=householder_q) -> np.ndarray:
    """ApproximatePCAEstimator.approximateQ (ApproximatePCA.scala:69-85, HMT Algorithm 4.4) with the test matrix given."""
    Q = qr(A @ omega)
    for _ in range(q):
        Qh = qr(A.T @ Q)
        Q = qr(A @ Qh)
    return Q


def approximate_pca(A: np.ndarray, omega: np.ndarray, dims: int, q: int, qr=householder_q) -> np.ndarray:
    """ApproximatePCAEstimator.approximatePCA (ApproximatePCA.scala:37-58): no centring; right singular vectors of B = Q^T A."""
    Q = approximate_q(A, omega, q, qr)
    _, _, vt = np.linalg.svd(Q.T @ A, full_matrices=False)
    return sign_convention(vt.T)[:, :dims]


def omega(d: int, l: int, seed: int = 0) -> np.ndarray:
    """The test matrix ApproximatePCAEstimator draws for this seed."""
    return np.random.default_rng(seed).standard_normal((d, l))


def zca_fit(X: np.ndarray, eps: float):
    """ZCAWhitenerEstimator.fitSingle (ZCAWhitener.scala:37-72) in fp64: (whitener, means)."""
    means = X.mean(0)
    _, s, vt = np.linalg.svd(X - means, full_matrices=False)  # N >= d
    s2 = s ** 2 / (X.shape[0] - 1.0)
    return vt.T @ np.diag((s2 + eps) ** -0.5) @ vt, means


def zca_apply(X: np.ndarray, whitener: np.ndarray, means: np.ndarray) -> np.ndarray:
    return (X - means) @ whitener


def pca_cost(n, d, k, sparsity, num_machines, cpu_weight, mem_weight, network_weight) -> float:
    """PCAEstimator.cost (PCA.scala:211-224)."""
    flops = float(n) * d * d
    return max(cpu_weight * flops, mem_weight * float(n) * d) + network_weight * float(n) * d


def distributed_pca_cost(n, d, k, sparsity, num_machines, cpu_weight, mem_weight, network_weight) -> float:
    """DistributedPCAEstimator.cost (DistributedPCA.scala:59-73)."""
    log2m = math.log(num_machines) / math.log(2.0)
    flops = float(n) * d * d / num_machines + float(d) * d * d * log2m
    return max(cpu_weight * flops, mem_weight * float(n) * d) + network_weight * float(d) * d * log2m


def planted(n: int, d: int, dims: int, rng: np.random.Generator, mean_scale: float = 3.0) -> np.ndarray:
    """Rows with a planted spectrum: the leading dims + 1 component scales fall by 5% each (about 10% gaps between eigenvalues),
    the rest are small; a random rotation and a non-zero column mean.  Returned as fp32 values in fp64."""
    k = dims + 1
    scales = np.concatenate([3.0 * 0.95 ** np.arange(k), np.full(d - k, 0.3 * 0.95 ** k)])
    rot = np.linalg.qr(rng.standard_normal((d, d)))[0]
    X = (rng.standard_normal((n, d)) * scales) @ rot.T + mean_scale * rng.standard_normal(d)
    return X.astype(np.float32).astype(np.float64)


def off_diagonal_cov(Y: np.ndarray) -> float:
    c = np.cov(Y, rowvar=False)
    return float(np.abs(c - np.diag(np.diag(c))).max())
