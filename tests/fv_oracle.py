"""fp64 NumPy oracle of the LCS Fisher-vector branch (K/nodes/images/{LCSExtractor,FisherVector}.scala,
K/nodes/learning/GaussianMixtureModel.scala, K/nodes/stats/{NormalizeRows,SignedHellingerMapper}.scala).

Layouts follow the reference: an LCS item is (n^2 C 2) x nKP (descriptors are columns), a GMM is means / variances D x K and K
weights, a Fisher vector is D x 2K.  The one deliberate deviation is fv2's last term, taken from Sanchez et al. (DESIGN.md section 16)."""
import math

import numpy as np


def _neighbours(s: int):
    return list(range(-2 * s + s // 2 - 1, s + s // 2 - 1 + 1, s))


def _keypoints(dim: int, start: int, stride: int):
    return list(range(start, dim - start, stride))


def box_stats(chan: np.ndarray, s: int):
    """ImageUtils.conv2D of one channel with the length-s box filter 1/s in both directions (zeros outside the image), for the
    values and their squares: window of (x, y) = rows [x - lo, x - lo + s), columns [y - lo, y - lo + s), lo = floor((s - 1) / 2).
    Returns (mean, sqrt(max(E[v^2] - mean^2, 0)))."""
    X, Y = chan.shape
    lo = (s - 1) // 2
    out = []
    for v in (chan, chan * chan):
        P = np.zeros((X + s - 1, Y + s - 1))
        P[lo:lo + X, lo:lo + Y] = v
        rows = sum(P[a:a + X, :] for a in range(s))
        out.append(sum(rows[:, b:b + Y] for b in range(s)) / (s * s))
    mean, sq = out
    return mean, np.sqrt(np.maximum(sq - mean * mean, 0.0))


def lcs_extract(img: np.ndarray, stride: int, stride_start: int, sub_patch_size: int, as_float: bool = True) -> np.ndarray:
    """LCSExtractor(stride, strideStart, subPatchSize).apply on img[x, y, c] (x = row): the (n^2 C 2) x nKP descriptor matrix, column
    xk * numPoolsY + yk, row ((c * n + nx) * n + ny) * 2 + {mean, std}; rounded to fp32 like the reference's Float output."""
    img = np.asarray(img, dtype=np.float64)
    X, Y, C = img.shape
    kx, ky, nb = _keypoints(X, stride_start, stride), _keypoints(Y, stride_start, stride), _neighbours(sub_patch_size)
    nn = len(nb)
    out = np.zeros((nn * nn * C * 2, len(kx) * len(ky)))
    for c in range(C):
        mean, std = box_stats(img[:, :, c], sub_patch_size)
        for a, ox in enumerate(nb):
            for b, oy in enumerate(nb):
                r = ((c * nn + a) * nn + b) * 2
                xs = np.asarray(kx)[:, None] + ox
                ys = np.asarray(ky)[None, :] + oy
                out[r] = mean[xs, ys].reshape(-1)
                out[r + 1] = std[xs, ys].reshape(-1)
    return out.astype(np.float32).astype(np.float64) if as_float else out


def gmm_posteriors(X: np.ndarray, means: np.ndarray, variances: np.ndarray, weights: np.ndarray, weight_threshold: float = 1e-4):
    """GaussianMixtureModel.apply(X) (GaussianMixtureModel.scala:47-82), X N x D, means / variances D x K: the reference's expanded
    Mahalanobis form, max shift, exp, normalise, threshold (keep > weightThreshold), normalise."""
    X = np.asarray(X, dtype=np.float64)
    mu, var, w = np.asarray(means, dtype=np.float64).T, np.asarray(variances, dtype=np.float64).T, np.asarray(weights, dtype=np.float64)
    D = X.shape[1]
    sq_mahl = (X * X) @ (0.5 / var).T - X @ (mu / var).T + 0.5 * (mu * mu / var).sum(1)[None, :]
    llh = (-0.5 * D * math.log(2 * math.pi) - 0.5 * np.log(var).sum(1) + np.log(w))[None, :] - sq_mahl
    llh = np.exp(llh - llh.max(1, keepdims=True))
    llh /= llh.sum(1, keepdims=True)
    t = np.where(llh > weight_threshold, llh, 0.0)
    return t / t.sum(1, keepdims=True)


def fisher_vector(x_item: np.ndarray, means, variances, weights, weight_threshold: float = 1e-4) -> np.ndarray:
    """FisherVector(gmm).apply on one item x_item (D x n): the D x 2K matrix [fv1 | fv2] with s0 = mean(q), s1 = X q / n,
    s2 = (X o X) q / n, fv1 = (s1 - mu diag(s0)) / (sigma diag(sqrt w)), fv2 = (s2 - 2 mu o s1 + (mu o mu - var) diag(s0)) /
    (var diag(sqrt(2 w)))."""
    x = np.asarray(x_item, dtype=np.float64)
    mu, var, w = (np.asarray(a, dtype=np.float64) for a in (means, variances, weights))
    n = x.shape[1]
    q = gmm_posteriors(x.T, mu, var, w, weight_threshold)
    s0 = q.mean(0)
    s1 = x @ q / n
    s2 = (x * x) @ q / n
    fv1 = (s1 - mu * s0[None, :]) / (np.sqrt(var) * np.sqrt(w)[None, :])
    fv2 = (s2 - 2.0 * mu * s1 + (mu * mu - var) * s0[None, :]) / (var * np.sqrt(2.0 * w)[None, :])
    return np.concatenate([fv1, fv2], 1)


def matrix_vectorizer(m: np.ndarray) -> np.ndarray:
    """MatrixVectorizer: column-major flattening, element (d, j) at d + D j."""
    return np.asarray(m).reshape(-1, order="F")


def normalize_rows(v: np.ndarray) -> np.ndarray:
    """NormalizeRows: each row divided by max(|row|_2, 2.2e-16)."""
    v = np.atleast_2d(np.asarray(v, dtype=np.float64))
    return v / np.maximum(np.sqrt((v * v).sum(1, keepdims=True)), 2.2e-16)


def signed_hellinger(v: np.ndarray) -> np.ndarray:
    """(Batch)SignedHellingerMapper: sign(v) sqrt(|v|)."""
    v = np.asarray(v, dtype=np.float64)
    return np.sign(v) * np.sqrt(np.abs(v))


def fv_tail(items, means, variances, weights, weight_threshold: float = 1e-4) -> np.ndarray:
    """The LCS branch after BatchPCATransformer: FisherVector -> FloatToDouble -> MatrixVectorizer -> NormalizeRows ->
    SignedHellingerMapper -> NormalizeRows, one row per item (items: PCA-projected descriptor matrices, dim x n_i)."""
    rows = []
    for it in items:
        fv = matrix_vectorizer(fisher_vector(it, means, variances, weights, weight_threshold))
        rows.append(normalize_rows(signed_hellinger(normalize_rows(fv)))[0])
    return np.stack(rows)
