"""fp64 NumPy restatement of what bwls.cu assembles for BlockWeightedLeastSquaresEstimator, and the per-class systems of the
reference semantics (K/nodes/learning/BlockWeightedLeastSquares.scala:241-273, K/ = src/main/scala/keystoneml/ of the reference
project) that the device's assembled systems are checked against.  Host code, no GPU.

The device never forms the raw-feature moments of the reference.  For each feature block it shifts the features by a vector m
(the exact population mean of materialised features, a sampled estimate for generated ones), and keeps only statistics of the
shifted block S = F - 1 m^T:
  * per class row range: the Gram S_c^T S_c, the column sums of S_c, S_c^T r_c (r_c: the class's own residual column) and
    the residual column sums over the class's rows;
  * over all rows: the sum of the class Grams, S^T R and the residual column sums.
`device_assembly_fit` rebuilds H, rhs and finalB from exactly these, in the order of bwls_build_kernel, bwls_rhs_kernel,
bwls_final_b_kernel and final_b_finish_kernel, so that it equals `keystone_oracle.bwls_fit` for ANY m up to fp64 rounding:
the shift is algebra, not an approximation.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np

from oracle import keystone_oracle as ko


def class_ranges(labels: np.ndarray):
    """Stable class sort of the rows (groupByClasses) and the (class, offset, count) runs of the present classes."""
    cls = np.argmax(np.asarray(labels), axis=1)
    perm = np.argsort(cls, kind="stable")
    counts = np.bincount(cls, minlength=labels.shape[1])
    ranges, off = [], 0
    for c in range(labels.shape[1]):
        if counts[c] > 0:
            ranges.append((c, off, int(counts[c])))
        off += int(counts[c])
    return perm, ranges


def device_assembly_fit(features: np.ndarray, labels: np.ndarray, block_size: int, num_iter: int, lam: float, w: float,
                        shift: Callable[[np.ndarray], np.ndarray], num_features: Optional[int] = None):
    """BlockWeightedLeastSquares as bwls.cu computes it, in fp64.  ``shift(block)`` returns the block's shift vector m (called
    once per block, at the first sweep, with the class-sorted block).  Returns ``(xs, final_b, systems)``; systems[(j, c)] =
    (H, rhs) of block j, class c at the first sweep."""
    perm, ranges = class_ranges(labels)
    F = np.asarray(features, dtype=np.float64)[perm]
    Y = np.asarray(labels, dtype=np.float64)[perm]
    n, k = Y.shape
    d = F.shape[1] if num_features is None else int(num_features)
    bounds = ko.block_bounds(d, block_size)
    counts = np.zeros(k)
    for c, _, nc in ranges:
        counts[c] = nc
    jlm = np.where(counts > 0, 2 * w + 2 * (1.0 - w) * counts / n - 1, 0.0)
    R = Y - jlm                                                    # bwls_init_residual_kernel
    xs = [np.zeros((e - s, k)) for s, e in bounds]
    shifts: List[Optional[np.ndarray]] = [None] * len(bounds)
    jms = [np.zeros((k, e - s)) for s, e in bounds]                # joint means, row per class
    systems = {}
    for it in range(num_iter):
        for j, (s0, e0) in enumerate(bounds):
            if it == 0:
                shifts[j] = np.asarray(shift(F[:, s0:e0]), dtype=np.float64)
            m = shifts[j]
            S = F[:, s0:e0] - m
            b = S.shape[1]
            # statistics of the shifted block
            rsum_all = R.sum(axis=0)
            psum = S.sum(axis=0)
            Gcls = [S[o:o + nc].T @ S[o:o + nc] for _, o, nc in ranges]
            Gpop = sum(Gcls)
            Cpop = S.T @ R
            dp = psum / n                                           # bwls_means_kernel
            dW = np.zeros((b, k))
            for (c, o, nc), Gc in zip(ranges, Gcls):
                Sc = S[o:o + nc]
                dc = Sc.sum(axis=0) / nc
                xtr = Sc.T @ R[o:o + nc, c]
                rsum_cls = R[o:o + nc].sum(axis=0)
                # bwls_build_kernel
                pop = Gpop / n - np.outer(dp, dp)
                cov = Gc / nc - np.outer(dc, dc)
                md = np.outer(dc - dp, dc - dp)
                H = (1.0 - w) * pop + w * cov + w * (1.0 - w) * md + lam * np.eye(b)
                # bwls_rhs_kernel: raw-feature F^T r = S^T r + m sum(r)
                pop_xtr = (Cpop[:, c] + m * rsum_all[c]) / n
                cls_xtr = (xtr + m * rsum_cls[c]) / nc
                joint_mean = m + w * dc + (1.0 - w) * dp
                mix = (rsum_all[c] / n) * (1.0 - w) + w * (rsum_cls[c] / nc)
                rhs = (1.0 - w) * pop_xtr + w * cls_xtr - joint_mean * mix - lam * xs[j][:, c]
                if it == 0:
                    jms[j][c] = joint_mean
                    systems[(j, c)] = (H, rhs)
                dW[:, c] = np.linalg.solve(H, rhs)
            xs[j] = xs[j] + dW
            R = R - (S @ dW + m @ dW)                               # R -= F dW = S dW + 1 (m^T dW)
    acc = sum((jm * x.T).sum(axis=1) for jm, x in zip(jms, xs))    # bwls_final_b_kernel
    return xs, jlm - acc, systems                                   # final_b_finish_kernel


def reference_systems(features: np.ndarray, labels: np.ndarray, block_size: int, lam: float, w: float, block: int,
                      num_features: Optional[int] = None, classes=None):
    """{class: (jointXTX + lambda I, jointXTR)} of feature block `block` at the first sweep, straight from the reference's
    definitions on raw features (BlockWeightedLeastSquares.scala:197-273).  jointXTR is the right-hand side of the block only
    for block 0, where the residual is still labels - jointLabelMean.  `classes`: only these (default: every present class)."""
    F = np.asarray(features, dtype=np.float64)
    Y = np.asarray(labels, dtype=np.float64)
    n, k = Y.shape
    cls = np.argmax(Y, axis=1)
    counts = np.bincount(cls, minlength=k)
    jlm = np.where(counts > 0, 2 * w + 2 * (1.0 - w) * counts / n - 1, 0.0)
    R = Y - jlm
    d = F.shape[1] if num_features is None else int(num_features)
    s0, e0 = ko.block_bounds(d, block_size)[block]
    A = F[:, s0:e0]
    pop_mean = A.mean(axis=0)
    pop_cov = A.T @ A / n - np.outer(pop_mean, pop_mean)
    pop_xtr = A.T @ R / n
    rmean = R.mean(axis=0)
    out = {}
    for c in (np.nonzero(counts)[0] if classes is None else classes):
        f = A[cls == c]
        r = R[cls == c, c]
        cm = f.mean(axis=0)
        zm = f - cm
        class_cov = zm.T @ zm / len(f)
        md = cm - pop_mean
        xtx = pop_cov * (1.0 - w) + class_cov * w + np.outer(md, md) * (1.0 - w) * w
        jm = cm * w + pop_mean * (1.0 - w)
        xtr = pop_xtr[:, c] * (1.0 - w) + (f.T @ r / len(f)) * w - jm * (rmean[c] * (1.0 - w) + w * r.mean())
        out[int(c)] = (xtx + lam * np.eye(e0 - s0), xtr)
    return out


def cond_bound(features: np.ndarray, labels: np.ndarray, block_size: int, lam: float, w: float,
               num_features: Optional[int] = None) -> float:
    """An upper bound on the largest 2-norm condition number of the per-class systems jointXTX + lambda I over all blocks (the
    systems do not change with the sweep).  jointXTX is a sum of positive semidefinite terms, so per class
      lambda_min >= (1 - w) lambda_min(popCov) + lambda,
      lambda_max <= (1 - w) lambda_max(popCov) + w lambda_max(classCov) + w (1 - w) |meanDiff|^2 + lambda;
    lambda_max(classCov) comes from the smaller of the two Gram orders of the centred class rows, which keeps this cheap
    at hundreds of classes."""
    F = np.asarray(features, dtype=np.float64)
    cls = np.argmax(np.asarray(labels), axis=1)
    d = F.shape[1] if num_features is None else int(num_features)
    worst = 0.0
    for s0, e0 in ko.block_bounds(d, block_size):
        A = F[:, s0:e0]
        pm = A.mean(axis=0)
        Z = A - pm
        ev = np.linalg.eigvalsh(Z.T @ Z / len(A))
        lo = (1.0 - w) * max(ev[0], 0.0) + lam
        for c in np.unique(cls):
            f = A[cls == c]
            zm = f - f.mean(axis=0)
            g = zm @ zm.T if len(f) < zm.shape[1] else zm.T @ zm
            cmax = np.linalg.eigvalsh(g)[-1] / len(f)
            md = f.mean(axis=0) - pm
            hi = (1.0 - w) * ev[-1] + w * cmax + w * (1.0 - w) * (md @ md) + lam
            worst = max(worst, hi / lo)
    return worst
