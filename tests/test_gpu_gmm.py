"""GaussianMixtureModelEstimator, KMeansPlusPlusEstimator / KMeansModel, GMMFisherVectorEstimator and ColumnSampler on the H100,
against the fp64 oracle (tests/gmm_oracle.py) fed the same fp32 samples and the same uniforms.

The shapes are N = 2e5 rows for (D, K) in {(3, 2), (64, 16)} and K = 1, and 5e4 rows at (80, 256).

Gates: identical k-means++ seed rows and Lloyd assignments, k-means means within 1e-12 relative; for EM the same iteration count and
stop reason, the cost history within 1e-12 relative per iteration, and means, variances and weights within 1e-9 relative Frobenius.
The device takes the Mahalanobis term in the direct form and the oracle in the reference's expanded form, so the only expected
difference is a posterior within rounding of weightThreshold; the synthetic mixtures are separated well enough that none is."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import KeystoneError, check, lib

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fv_oracle as fo  # noqa: E402
import gmm_oracle as go  # noqa: E402
import pca_oracle as po  # noqa: E402

pytestmark = pytest.mark.gpu
KS_ERR_INVALID = -1
N = 200_000


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


def _rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(np.asarray(a) - b) / max(np.linalg.norm(b), 1e-300))


def _rows(K):
    """N rows, and 5e4 at K = 256: there the fp64 oracle's k-means++ and assignments (sums over d in order, as the device) take
    minutes per fit on the host."""
    return N if K < 256 else 50_000


def _sample(D, K, seed):
    """Well-separated clusters; at K = 256 overlapping ones, because k-means++ on 256 separated clusters empties some (see
    test_rejections)."""
    return go.mixture_sample(_rows(K), D, K, seed=seed, spread=1.0 if K >= 256 else 6.0)


def _dm(ctx, X):
    return ctx.matrix(np.asarray(X, dtype=np.float32))


@pytest.mark.parametrize("D,K,iters", [(3, 2, 20), (64, 16, 4), (80, 256, 2), (5, 1, 3)])
def test_kmeans_matches_oracle(ctx, D, K, iters):
    X = _sample(D, K, D + K)
    est = ks.KMeansPlusPlusEstimator(K, iters)
    model = est.fit(_dm(ctx, X))
    ref = go.kmeans_fit(X, K, iters, 1e-3, est.uniforms())
    assert list(est.seed_rows) == list(ref["seeds"])
    assert est.stats["solver"] == "kmeans" and est.stats["iterations"] == ref["iterations"]
    assert _rel(model.means, ref["means"]) <= 1e-12
    np.testing.assert_allclose(est.stats["cost_history"], ref["costs"], rtol=1e-12)
    got = model.apply(_dm(ctx, X)).to_numpy()
    idx, _ = go.assign(X, model.means)
    assert (got.sum(1) == 1).all() and np.array_equal(got.argmax(1), idx)


CASES = [  # D, K, init, estimator keywords, expected stop reason
    (3, 2, "kmeans++", dict(maxIterations=100), "cost"),
    (64, 16, "kmeans++", dict(maxIterations=4, stopTolerance=-1.0), "max_iterations"),
    (80, 256, "kmeans++", dict(maxIterations=2, minClusterSize=1, stopTolerance=-1.0), "max_iterations"),
    (5, 1, "kmeans++", dict(maxIterations=3), None),
    (3, 2, "random", dict(maxIterations=100), None),
    (8, 4, "random", dict(maxIterations=6), None),
    (3, 3, "kmeans++", dict(maxIterations=100, minClusterSize=N // 3 + 2000), "min_cluster_size"),
]


@pytest.mark.parametrize("D,K,init,kw,reason", CASES)
def test_gmm_matches_oracle(ctx, D, K, init, kw, reason):
    X = _sample(D, K, 10 * D + K)
    meth = ks.KMEANS_PLUS_PLUS_INITIALIZATION if init == "kmeans++" else ks.RANDOM_INITIALIZATION
    est = ks.GaussianMixtureModelEstimator(K, initializationMethod=meth, **kw)
    gmm = est.fit(_dm(ctx, X))
    u = est.uniforms(D)
    ref = go.gmm_fit(X, K, max_iterations=kw["maxIterations"], min_cluster_size=kw.get("minClusterSize", 40),
                     stop_tolerance=kw.get("stopTolerance", 1e-4), init=init, uniforms=u)
    st = est.stats
    assert st["solver"] == "gmm" and (st["n"], st["d"], st["k"]) == (_rows(K), D, K)
    assert st["stop_reason"] == ref["stop_reason"] and reason in (None, ref["stop_reason"])
    assert st["iterations"] == ref["iterations"]
    if init == "kmeans++":
        assert st["seed_rows"] == list(ref["seeds"])
    np.testing.assert_allclose(st["cost_history"], ref["costs"], rtol=1e-12)
    assert _rel(gmm.means, ref["means"]) <= 1e-9
    assert _rel(gmm.variances, ref["variances"]) <= 1e-9
    assert _rel(gmm.weights, ref["weights"]) <= 1e-9
    assert gmm.weight_threshold == 1e-4
    # the returned handle is the model: its posteriors equal those of a model re-created from the host arrays
    again = ks.GaussianMixtureModel(gmm.means, gmm.variances, gmm.weights, ctx=ctx)
    x = _dm(ctx, X[:4096])
    assert np.array_equal(gmm.apply(x).to_numpy(), again.apply(x).to_numpy())


def test_repeated_fit_is_bit_identical(ctx):
    X = _dm(ctx, go.mixture_sample(N, 64, 16, seed=5))
    fits = [ks.GaussianMixtureModelEstimator(16, maxIterations=5).fit(X) for _ in range(2)]
    for a in ("means", "variances", "weights"):
        assert np.array_equal(getattr(fits[0], a), getattr(fits[1], a))
    km = [ks.KMeansPlusPlusEstimator(16, 3).fit(X).means for _ in range(2)]
    assert np.array_equal(km[0], km[1])


DATA1 = np.array([[1.0, 2.0, 6.0], [1.0, 3.0, 0.0], [1.0, 4.0, 6.0], [1.0, 1.0, 0.0]])
MLLIB = np.array([-5.1971, -2.5359, -3.8220, -5.2211, -5.0602, 4.7118, 6.8989, 3.4592, 4.6322, 5.7048, 4.6567, 5.5026, 4.5605, 5.2043,
                  6.2734])[:, None]


def test_reference_suites_on_device(ctx):
    """GaussianMixtureModelSuite and KMeansPlusPlusSuite through the device nodes (default seed)."""
    g = ks.GaussianMixtureModelEstimator(1, minClusterSize=1, ctx=ctx).fit(DATA1[:3])
    assert np.array_equal(g.means.T, [[1.0, 3.0, 4.0]])
    g = ks.GaussianMixtureModelEstimator(2, minClusterSize=1, ctx=ctx).fit(DATA1)
    assert {tuple(r) for r in g.means.T} == {(1.0, 2.0, 0.0), (1.0, 3.0, 6.0)}
    assert {tuple(r) for r in g.variances.T} == {(1e-9, 1.0, 0.09)}
    g = ks.GaussianMixtureModelEstimator(2, minClusterSize=1, ctx=ctx).fit(MLLIB)
    order = np.argsort(-g.means[0])
    assert np.allclose(g.means[0][order], [5.1604, -4.3673], atol=1e-4)
    assert np.allclose(g.variances[0][order], [0.86644, 1.1098], atol=1e-4)
    data3 = np.loadtxt(os.path.join(HERE, "golden", "gmm_data.txt"))
    g = ks.GaussianMixtureModelEstimator(2, minClusterSize=1, stopTolerance=0, maxIterations=30, ctx=ctx).fit(data3)
    assert np.abs(g.means).max() <= 0.5
    v = g.variances
    assert np.abs(v - [[1.0, 25.0], [25.0, 1.0]]).max() <= 2.0 or np.abs(v - [[25.0, 1.0], [1.0, 25.0]]).max() <= 2.0
    assert np.abs(g.weights - 0.5).max() <= 0.05
    for it in (1, 10):
        assert np.allclose(ks.KMeansPlusPlusEstimator(1, it, ctx=ctx).fit(DATA1[:3]).means, [[1.0, 3.0, 4.0]])
    for it in (10, 5):
        assert {tuple(r) for r in ks.KMeansPlusPlusEstimator(2, it, ctx=ctx).fit(DATA1).means} == {(1.0, 2.0, 0.0), (1.0, 3.0, 6.0)}
    km = ks.KMeansModel(np.array([[1.0, 2.0, 0.0], [1.0, 3.0, 6.0]]), ctx=ctx)
    assert np.array_equal(km.apply(DATA1).to_numpy(), [[0, 1], [1, 0], [0, 1], [1, 0]])
    assert np.array_equal(km.apply(np.array([1.0, 3.0, 0.0])), [1.0, 0.0])


def _gmm_fit_rc(ctx, x, k, thr=1e-4, init=0, u=None, dim=1):
    u = np.ascontiguousarray(np.full(k * (dim if init else 1), 0.5) if u is None else u, dtype=np.float64)
    kk = max(k, 1)
    m, v, w = np.zeros(kk * dim), np.zeros(kk * dim), np.zeros(kk)
    h = C.c_int64(0)
    rc = lib().ks_gmm_fit(ctx.handle, x.handle, k, 10, 1.0, 1e-4, thr, 1e-2, 1e-9, init, u.ctypes.data_as(C.c_void_p), C.byref(h),
                          m.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p), None)
    return rc, (lib().ks_last_error(ctx.handle) or b"").decode()


def test_rejections(ctx):
    X = go.mixture_sample(1000, 3, 2, seed=9)
    x = _dm(ctx, X)
    for args, needle in [((0,), "centres"), ((1001,), "fewer rows"), ((4, 0.25), "weightThreshold"), ((2, 1e-4, 0, [0.5, 1.0]), "[0, 1)")]:
        rc, msg = _gmm_fit_rc(ctx, x, *args, dim=3)
        assert rc == KS_ERR_INVALID and needle in msg, (args, msg)
    rc, msg = _gmm_fit_rc(ctx, _dm(ctx, np.zeros((4, 1100))), 2, dim=1100)
    assert rc == KS_ERR_INVALID and "1024" in msg
    bad = X.copy()
    bad[17, 1] = np.nan
    rc, msg = _gmm_fit_rc(ctx, _dm(ctx, bad), 2, dim=3)
    assert rc == KS_ERR_INVALID and "non-finite" in msg
    rc, msg = _gmm_fit_rc(ctx, _dm(ctx, np.tile([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]], (50, 1))), 3, dim=3)
    assert rc == KS_ERR_INVALID and "distinct" in msg
    for est in (ks.KMeansPlusPlusEstimator(3, 2), ks.GaussianMixtureModelEstimator(3)):
        with pytest.raises(KeystoneError, match="distinct"):
            est.fit(_dm(ctx, np.tile([[1.0, 2.0]], (10, 1))))
    # k-means++ at the default seed on 256 separated clusters leaves cluster 63 empty in the second Lloyd pass (seed-dependent; the
    # oracle agrees); the reference returns NaN means there
    sep = _dm(ctx, go.mixture_sample(N, 80, 256, seed=336))
    with pytest.raises(KeystoneError, match="cluster 63 is empty") as e:
        ks.KMeansPlusPlusEstimator(256, 2).fit(sep)
    assert e.value.code == KS_ERR_INVALID
    with pytest.raises(KeystoneError, match="cluster 63 is empty"):
        ks.GaussianMixtureModelEstimator(256).fit(sep)
    with pytest.raises(KeystoneError) as e:  # means of another dimension
        ks.KMeansModel(np.zeros((2, 2)), ctx=ctx).apply(np.zeros((3, 3)))
    assert e.value.code == KS_ERR_INVALID


def test_column_sampler_gathers_host_rows(ctx):
    rng = np.random.default_rng(3)
    items = [rng.standard_normal((6, n)).astype(np.float32) for n in (5, 17, 1, 40)]
    batch = ks.ItemBatch.from_items(ctx, items)
    s = ks.ColumnSampler(7, seed=11)
    out = s.apply(batch)
    rows = ks.ColumnSampler(7, seed=11).sample_rows(batch.offsets)
    assert np.array_equal(out.offsets, np.arange(5) * 7)
    assert np.array_equal(out.to_numpy(np.float32), batch.to_numpy(np.float32)[rows])
    for i, it in enumerate(out.to_list()):
        cols = rows[7 * i:7 * (i + 1)] - batch.offsets[i]
        assert ((cols >= 0) & (cols < items[i].shape[1])).all()
        assert np.array_equal(it, items[i][:, cols].astype(np.float64))


def test_miniature_fisher_branch_end_to_end(ctx):
    """LCSExtractor -> ColumnSampler -> ColumnPCAEstimator / BatchPCATransformer -> GMMFisherVectorEstimator.fit -> FisherVector ->
    NormalizeRows -> SignedHellingerMapper -> NormalizeRows, against fv_oracle.fv_tail with the GMM the oracle fits from the same
    sample."""
    rng = np.random.default_rng(21)
    imgs = (rng.random((64, 32, 32, 3)) * 255).astype(np.float32)
    lcs = ks.LCSExtractor(4, 8, 4).apply(ks.ImageBatch.from_images(ctx, imgs))
    sample = ks.ColumnSampler(40, seed=1).apply(lcs)
    pca = ks.ColumnPCAEstimator(8, ctx=ctx).fit(sample.to_list(np.float32))
    zs = pca.apply(sample)
    est = ks.GMMFisherVectorEstimator(4, ctx=ctx)
    fv = est.fit(zs)
    zrows = zs.matrix.to_numpy()
    ref = go.gmm_fit(zrows, 4, uniforms=est.gmm_estimator.uniforms(8))
    assert est.gmm_estimator.stats["iterations"] == ref["iterations"]
    assert _rel(fv.gmm.means, ref["means"]) <= 1e-9 and _rel(fv.gmm.variances, ref["variances"]) <= 1e-9
    z = pca.apply(lcs)
    F = ks.Pipeline([fv, ks.FloatToDouble(), ks.MatrixVectorizer(), ks.NormalizeRows(), ks.SignedHellingerMapper(), ks.NormalizeRows()])(z)
    F = F.to_numpy()
    tail = fo.fv_tail(z.to_list(), ref["means"], ref["variances"], ref["weights"])
    for i in range(F.shape[0]):
        assert _rel(F[i], tail[i]) <= 1e-5, (i, _rel(F[i], tail[i]))
