"""fp64 NumPy oracle of Gaussian-kernel ridge regression: the reference semantics the device fit and apply are checked against.

GaussianKernelGenerator (K/nodes/learning/KernelGenerator.scala:121-194), KernelRidgeRegression.trainWithL2
(K/nodes/learning/KernelRidgeRegression.scala:86-235) and KernelBlockLinearMapper.apply (KernelBlockLinearMapper.scala:39-89),
K/ = src/main/scala/keystoneml/ of the reference project.  Host code, no GPU.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np


def gaussian_kernel(X: np.ndarray, Z: np.ndarray, gamma: float) -> np.ndarray:
    """K[i, j] = exp(-gamma |x_i - z_j|^2), computed as |x|^2 + |z|^2 - 2 x.z (KernelGenerator.scala:160-176)."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.asarray(Z, dtype=np.float64)
    xx = np.sum(X * X, axis=1)[:, None]
    zz = np.sum(Z * Z, axis=1)[None, :]
    return np.exp(-gamma * (xx + zz - 2.0 * X @ Z.T))


def block_ranges(n: int, block_size: int):
    """Contiguous blocks of training rows, the last one ragged (KernelRidgeRegression.scala:101, 143)."""
    nb = -(-n // block_size)
    return [(j * block_size, min(n, (j + 1) * block_size)) for j in range(nb)]


def krr_fit(X: np.ndarray, Y: np.ndarray, gamma: float, lam: float, block_size: int, num_epochs: int,
            block_order: Optional[Sequence[Sequence[int]]] = None) -> List[np.ndarray]:
    """trainWithL2 in the reference form: per block, C = K_B^T W, rhs = Y_B - (C - K_BB^T W_B,old), W_B = (K_BB + lam I) \\ rhs
    (an LU solve there; numpy.linalg.solve here).  block_order[e] is epoch e's block order (None: sequential).  Returns the
    per-block weights W_j (b_j x k)."""
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    n = X.shape[0]
    blocks = block_ranges(n, block_size)
    W = np.zeros_like(Y)
    for e in range(num_epochs):
        order = range(len(blocks)) if block_order is None else block_order[e]
        for j in order:
            lo, hi = blocks[j]
            KB = gaussian_kernel(X, X[lo:hi], gamma)             # n x b
            KBB = KB[lo:hi]                                      # diagBlock
            C = KB.T @ W
            w_old = W[lo:hi] if e > 0 else np.zeros((hi - lo, Y.shape[1]))
            rhs = Y[lo:hi] - (C - KBB.T @ w_old)
            W[lo:hi] = np.linalg.solve(KBB + lam * np.eye(hi - lo), rhs)
    return [W[lo:hi].copy() for lo, hi in blocks]


def kernel_block_apply(X_test: np.ndarray, X_train: np.ndarray, gamma: float, xs: Sequence[np.ndarray], block_size: int) -> np.ndarray:
    """KernelBlockLinearMapper.apply: sum_j K(X_test, X_train[block j]) W_j."""
    out = np.zeros((np.asarray(X_test).shape[0], np.asarray(xs[0]).shape[1]))
    for (lo, hi), w in zip(block_ranges(np.asarray(X_train).shape[0], block_size), xs):
        out += gaussian_kernel(X_test, np.asarray(X_train)[lo:hi], gamma) @ np.asarray(w, dtype=np.float64)
    return out
