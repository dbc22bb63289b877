"""The fp64 mixture / k-means oracle against the reference suites (GaussianMixtureModelSuite, KMeansPlusPlusSuite) and the EM loop's
semantics; CPU only.  Assertions hold at the nodes' default seed (0); a seed-dependent one says so."""
import os

import numpy as np
import pytest

import gmm_oracle as go

HERE = os.path.dirname(os.path.abspath(__file__))
DATA1 = np.array([[1.0, 2.0, 6.0], [1.0, 3.0, 0.0], [1.0, 4.0, 6.0], [1.0, 1.0, 0.0]])
MLLIB = np.array([-5.1971, -2.5359, -3.8220, -5.2211, -5.0602, 4.7118, 6.8989, 3.4592, 4.6322, 5.7048, 4.6567, 5.5026, 4.5605, 5.2043,
                  6.2734])[:, None]


def gmm_data():
    return np.loadtxt(os.path.join(HERE, "golden", "gmm_data.txt"))


def rows(m):
    return {tuple(r) for r in np.asarray(m)}


def test_gmm_single_centre_exact():
    r = go.gmm_fit(DATA1[:3], 1, min_cluster_size=1, uniforms=go.default_uniforms(1))
    assert np.array_equal(r["means"].T, [[1.0, 3.0, 4.0]])


def test_gmm_two_centres_dataset1_exact():
    r = go.gmm_fit(DATA1, 2, min_cluster_size=1, uniforms=go.default_uniforms(2))
    assert rows(r["means"].T) == {(1.0, 2.0, 0.0), (1.0, 3.0, 6.0)}
    assert rows(r["variances"].T) == {(1e-9, 1.0, 0.09)}


def test_gmm_two_centres_dataset2_mllib():
    r = go.gmm_fit(MLLIB, 2, min_cluster_size=1, uniforms=go.default_uniforms(2))
    m, v = r["means"][0], r["variances"][0]
    order = np.argsort(-m)
    assert np.allclose(m[order], [5.1604, -4.3673], atol=1e-4)
    assert np.allclose(v[order], [0.86644, 1.1098], atol=1e-4)


def test_gmm_two_centres_dataset3_file():
    r = go.gmm_fit(gmm_data(), 2, min_cluster_size=1, stop_tolerance=0, max_iterations=30, uniforms=go.default_uniforms(2))
    assert np.abs(r["means"]).max() <= 0.5
    v = r["variances"]
    assert np.abs(v - [[1.0, 25.0], [25.0, 1.0]]).max() <= 2.0 or np.abs(v - [[25.0, 1.0], [1.0, 25.0]]).max() <= 2.0
    assert np.abs(r["weights"] - 0.5).max() <= 0.05


def test_kmeans_single_centre():
    for it in (1, 10):
        r = go.kmeans_fit(DATA1[:3], 1, it, 1e-3, go.default_uniforms(1))
        assert np.allclose(r["means"], [[1.0, 3.0, 4.0]])


def test_kmeans_two_centres():
    for it in (10, 5):
        r = go.kmeans_fit(DATA1, 2, it, 1e-3, go.default_uniforms(2))
        assert rows(r["means"]) == {(1.0, 2.0, 0.0), (1.0, 3.0, 6.0)}


def test_kmeans_transformer():
    idx, _ = go.assign(DATA1, np.array([[1.0, 2.0, 0.0], [1.0, 3.0, 6.0]]))
    assert list(idx) == [1, 0, 1, 0]


def test_xerox_lse_cutoffs():
    llh = np.array([[0.0, 0.0, -100.0], [0.0, 40.0, 0.0], [-5.0, 1.0, 2.0]])
    lse = go.xerox_lse(llh)
    # a component more than 30 below adds no weight: lse = (lse - l) + l, exactly as the reference rounds it
    assert lse[0] == (np.log(2.0) + 100.0) - 100.0
    assert lse[1] == 40.0                              # delta -40 (below -30), then delta 40 (above 30)
    ref = np.log(np.exp(-5.0) + np.exp(1.0) + np.exp(2.0))
    assert abs(lse[2] - ref) < 1e-12


def test_draw_rule():
    d = np.zeros(600)
    d[[3, 300, 599]] = [1.0, 2.0, 1.0]
    assert go.draw_row(d, 0.0) == 3
    assert go.draw_row(d, 0.25) == 300        # C = 1 at row 3, 3 at row 300: first C > 1
    assert go.draw_row(d, 0.7499) == 300
    assert go.draw_row(d, 0.75) == 599
    with pytest.raises(ValueError):
        go.draw_row(np.zeros(10), 0.5)


def test_gmm_stop_on_cost_evaluates_estep_without_mstep():
    X = go.mixture_sample(4000, 3, 2, seed=1)
    full = go.gmm_fit(X, 2, max_iterations=100, uniforms=go.default_uniforms(2))
    assert full["stop_reason"] == "cost"
    n = full["iterations"]
    # the same fit capped one E-step earlier ends on max_iterations after its last M-step; the stopping E-step changes nothing
    capped = go.gmm_fit(X, 2, max_iterations=n - 1, uniforms=go.default_uniforms(2))
    assert capped["stop_reason"] == "max_iterations" and capped["costs"] == full["costs"][:-1]
    assert np.array_equal(capped["means"], full["means"]) and np.array_equal(capped["variances"], full["variances"])
    assert full["costs"][-1] - full["costs"][-2] < 1e-4 * abs(full["costs"][-2])


def test_gmm_small_cluster_keeps_previous_parameters():
    X = go.mixture_sample(2000, 3, 3, seed=2)
    stop = go.gmm_fit(X, 3, min_cluster_size=700, uniforms=go.default_uniforms(3))
    assert stop["stop_reason"] == "min_cluster_size"
    n = stop["iterations"]
    prev = go.gmm_fit(X, 3, min_cluster_size=1, max_iterations=n - 1, uniforms=go.default_uniforms(3)) if n > 1 else None
    if prev is not None:
        assert np.array_equal(prev["means"], stop["means"])
    else:  # stopped at the first E-step: the initialisation is returned
        init = go.gmm_fit(X, 3, min_cluster_size=1, max_iterations=1, uniforms=go.default_uniforms(3))
        assert init["iterations"] == 1


def test_returned_model_uses_default_threshold():
    r = go.gmm_fit(DATA1, 2, min_cluster_size=1, weight_threshold=0.3, uniforms=go.default_uniforms(2))
    assert r["weight_threshold"] == 1e-4


def test_random_initialisation():
    X = go.mixture_sample(3000, 2, 2, seed=3)
    r = go.gmm_fit(X, 2, init="random", uniforms=go.default_uniforms(2, 2, init="random"))
    assert r["seeds"] is None and np.isfinite(r["means"]).all() and abs(r["weights"].sum() - 1.0) < 1e-12
