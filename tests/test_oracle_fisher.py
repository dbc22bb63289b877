"""The fp64 oracle of the LCS Fisher-vector branch (tests/fv_oracle.py) against the reference's known answers and closed forms."""
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fv_oracle as fo  # noqa: E402
from oracle import keystone_oracle as ko  # noqa: E402


def gantrycrane(golden_dir):
    """images/gantrycrane.png as ImageUtils.loadImage yields it: channels in BGR order, x = row."""
    return ko.image_from_bgr_bytes(np.load(os.path.join(golden_dir, "conv_gantrycrane.npz"))["rgb"])


def test_lcs_matches_matlab_sums(golden_dir):
    """LCSExtractorSuite "Load an Image and compute LCS Features": (stride 4, subPatch 6, strideStart 16), MATLAB sums to 1e-8."""
    L = fo.lcs_extract(gantrycrane(golden_dir), 4, 16, 6)
    assert L.shape == (96, 5336)
    first, total = 3.786557667540610e+03, 3.171963632855949e+07
    assert abs(L[:, 0].sum() - first) / first < 1e-8
    assert abs(L.sum() - total) / total < 1e-8


def test_lcs_window_is_zero_padded_box():
    """A single bright pixel: the window mean is 1/s^2 exactly where the window [x - lo, x - lo + s) covers it."""
    img = np.zeros((40, 40, 1))
    img[20, 20, 0] = 1.0
    mean, std = fo.box_stats(img[:, :, 0], 6)
    rows, cols = np.nonzero(mean)
    assert rows.min() == 20 - 3 and rows.max() == 20 + 2 and cols.min() == 17 and cols.max() == 22   # lo = 2, hi = 3
    assert np.allclose(mean[rows, cols], 1 / 36) and np.allclose(std[rows, cols], math.sqrt(1 / 36 - 1 / 36 ** 2))


def test_gmm_known_answer():
    """GaussianMixtureModelSuite "GaussianMixtureModel test": exact one-hot posteriors with sigma^2 = 1e-8 in the first dimension."""
    data = np.array([[1.0, 2.0, 6.0], [1.0, 3.0, 0.0], [1.0, 4.0, 6.0], [1.0, 1.0, 0.0]])
    means = np.array([[1.0, 2.0, 0.0], [1.0, 3.0, 6.0]]).T
    variances = np.array([[1e-8, 1.0, 0.09], [1e-8, 1.0, 0.09]]).T
    q = fo.gmm_posteriors(data, means, variances, np.array([0.5, 0.5]))
    assert np.array_equal(q, np.array([[0.0, 1.0], [1.0, 0.0], [0.0, 1.0], [1.0, 0.0]]))


def test_posteriors_sum_to_one_after_threshold():
    rng = np.random.default_rng(0)
    D, K = 8, 16
    means, variances = rng.standard_normal((D, K)), rng.uniform(0.5, 2.0, (D, K))
    w = rng.uniform(0.5, 1.5, K)
    q = fo.gmm_posteriors(rng.standard_normal((500, D)) * 1.5, means, variances, w / w.sum(), 1e-2)
    assert np.allclose(q.sum(1), 1.0, atol=1e-14)
    assert ((q == 0) | (q > 1e-2)).all() and (q == 0).any()


def test_fisher_vector_single_component_closed_forms():
    """K = 1: every posterior is 1, so fv1 = (mean(x) - mu) / sigma and fv2 = (mean((x - mu)^2) - sigma^2) / (sigma^2 sqrt 2)."""
    rng = np.random.default_rng(1)
    D, n = 5, 37
    x = rng.standard_normal((D, n)) * 2 + 1
    mu, var = rng.standard_normal((D, 1)), rng.uniform(0.5, 3.0, (D, 1))
    fv = fo.fisher_vector(x, mu, var, np.array([1.0]))
    assert fv.shape == (D, 2)
    sig = np.sqrt(var[:, 0])
    assert np.allclose(fv[:, 0], (x.mean(1) - mu[:, 0]) / sig, rtol=1e-12, atol=1e-13)
    assert np.allclose(fv[:, 1], (((x - mu) ** 2).mean(1) - var[:, 0]) / (var[:, 0] * math.sqrt(2)), rtol=1e-12, atol=1e-13)


def test_fisher_vector_is_the_sanchez_form():
    """fv2 = sum_n q ((x - mu)^2 / sigma^2 - 1) / (n sqrt(2 w)) and fv1 = sum_n q (x - mu) / sigma / (n sqrt w), at D != K."""
    rng = np.random.default_rng(2)
    D, K, n = 3, 2, 11
    x = rng.standard_normal((D, n))
    mu, var = rng.standard_normal((D, K)) * 0.5, rng.uniform(0.5, 2.0, (D, K))
    w = np.array([0.3, 0.7])
    q = fo.gmm_posteriors(x.T, mu, var, w)
    fv = fo.fisher_vector(x, mu, var, w)
    for k in range(K):
        z = (x - mu[:, k:k + 1]) / np.sqrt(var[:, k:k + 1])
        assert np.allclose(fv[:, k], (z * q[:, k]).sum(1) / (n * math.sqrt(w[k])), atol=1e-13)
        assert np.allclose(fv[:, K + k], ((z * z - 1) * q[:, k]).sum(1) / (n * math.sqrt(2 * w[k])), atol=1e-13)


def test_normalize_rows_floor_and_signed_hellinger_signs():
    v = np.array([[3.0, -4.0, 0.0], [0.0, 0.0, 0.0], [1e-20, 0.0, 0.0]])
    out = fo.normalize_rows(v)
    assert np.allclose(out[0], [0.6, -0.8, 0.0]) and np.array_equal(out[1], np.zeros(3))
    assert out[2, 0] == 1e-20 / 2.2e-16   # the floor: a row shorter than 2.2e-16 is divided by 2.2e-16
    h = fo.signed_hellinger(np.array([-4.0, 0.0, 9.0, -0.25]))
    assert np.array_equal(h, [-2.0, 0.0, 3.0, -0.5])
    assert np.array_equal(fo.matrix_vectorizer(np.array([[1, 2], [3, 4]])), [1, 3, 2, 4])
