"""LCSExtractor, GaussianMixtureModel posteriors, FisherVector, NormalizeRows and the signed square root on the H100, against the fp64
oracle (tests/fv_oracle.py) on the same fp32 arrays, and the miniature LCS branch end to end into BlockWeightedLeastSquaresEstimator.

Gates: LCS to the reference's MATLAB sums (1e-8 relative) and 1e-4 absolute per element (a flat window makes the std a
cancellation); posteriors within 1e-12 of the fp64 oracle before their storage rounding to fp32, with the same entries thresholded
to zero; Fisher vectors (fp32 output) within 1e-6 relative Frobenius per item and bit-identical on a repeated call."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import check, lib
from oracle import keystone_oracle as ko

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import bwls_oracle as bo  # noqa: E402
import fv_oracle as fo  # noqa: E402
import pca_oracle as po  # noqa: E402

pytestmark = pytest.mark.gpu

W_TOL = 1e-4   # tests/test_gpu_bwls.py
KS_ERR_INVALID, KS_ERR_HANDLE = -1, -6


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


def _gmm(rng, D, K, spread=1.0):
    means = rng.standard_normal((D, K)) * spread
    variances = rng.uniform(0.5, 2.0, (D, K))
    w = rng.uniform(0.5, 1.5, K)
    return means, variances, w / w.sum()


# ---------------------------------------------------------------------------------------------------------------- LCS
def test_lcs_gantrycrane_matches_matlab(ctx, golden_dir):
    img = ko.image_from_bgr_bytes(np.load(os.path.join(golden_dir, "conv_gantrycrane.npz"))["rgb"])
    items = ks.LCSExtractor(4, 16, 6).apply(ks.ImageBatch.from_images(ctx, img[None]))
    assert items.n_items == 1 and items.matrix.shape == (5336, 96)
    L = items.to_list()[0]
    assert L.shape == (96, 5336)
    first, total = 3.786557667540610e+03, 3.171963632855949e+07
    assert abs(L[:, 0].sum() - first) / first < 1e-8
    assert abs(L.sum() - total) / total < 1e-8
    ref = fo.lcs_extract(img, 4, 16, 6)
    assert np.abs(L - ref).max() <= 1e-4, np.abs(L - ref).max()


@pytest.mark.parametrize("shape,stride,start,s", [((37, 53, 1), 3, 9, 4), ((48, 31, 3), 5, 12, 5), ((21, 26, 3), 2, 4, 2),
                                                  ((33, 33, 1), 1, 4, 1), ((40, 29, 3), 4, 10, 3)])
def test_lcs_synthetic_batches(ctx, shape, stride, start, s):
    rng = np.random.default_rng(sum(shape) * 31 + s)
    imgs = (rng.random((5,) + shape) * 255).astype(np.float32)
    items = ks.LCSExtractor(stride, start, s).apply(ks.ImageBatch.from_images(ctx, imgs))
    got = items.to_list()
    assert len(got) == 5
    for im, L in zip(imgs, got):
        ref = fo.lcs_extract(im.astype(np.float64), stride, start, s)
        assert L.shape == ref.shape
        assert np.abs(L - ref).max() <= 1e-4, np.abs(L - ref).max()


def test_lcs_list_of_mixed_shapes_keeps_order(ctx):
    rng = np.random.default_rng(3)
    shapes = [(36, 40, 3), (30, 30, 3), (36, 40, 3), (30, 30, 3), (36, 40, 3)]
    imgs = [(rng.random(sh) * 255).astype(np.float32) for sh in shapes]
    node = ks.LCSExtractor(4, 10, 3, ctx=ctx)
    got = node.apply(imgs).to_list()
    for im, L in zip(imgs, got):
        assert np.abs(L - fo.lcs_extract(im.astype(np.float64), 4, 10, 3)).max() <= 1e-4
    single = node.apply(imgs[1])
    assert single.dtype == np.float32 and np.array_equal(single.astype(np.float64), got[1])


def test_lcs_batch_spanning_several_launches(ctx):
    """300 images of 256 x 256 x 3 at the pipeline's settings: the window statistics are bounded to 16 MB per launch pair.  The
    keypoints use 118 distinct window centres per axis (3 x 118^2 float2 per image), so 50 images go in a pair: six pairs."""
    rng = np.random.default_rng(4)
    imgs = rng.integers(0, 256, (300, 256, 256, 3)).astype(np.float32)
    batch = ks.ImageBatch.from_images(ctx, imgs)
    l0 = ctx.launch_count()
    items = ks.LCSExtractor(4, 16, 6).apply(batch)
    assert ctx.launch_count() - l0 == 12
    assert items.n_items == 300 and items.matrix.shape == (300 * 3136, 96)
    host = items.matrix.to_numpy()
    for i in (0, 49, 50, 299):
        ref = fo.lcs_extract(imgs[i].astype(np.float64), 4, 16, 6)
        assert np.abs(host[i * 3136:(i + 1) * 3136].T - ref).max() <= 1e-4


# ---------------------------------------------------------------------------------------------------------------- posteriors
def test_gmm_known_answer(ctx):
    """GaussianMixtureModelSuite "GaussianMixtureModel test": exact one-hot posteriors, vector and matrix apply."""
    data = np.array([[1.0, 2.0, 6.0], [1.0, 3.0, 0.0], [1.0, 4.0, 6.0], [1.0, 1.0, 0.0]])
    means = np.array([[1.0, 2.0, 0.0], [1.0, 3.0, 6.0]]).T
    variances = np.array([[1e-8, 1.0, 0.09], [1e-8, 1.0, 0.09]]).T
    gmm = ks.GaussianMixtureModel(means, variances, np.array([0.5, 0.5]), ctx=ctx)
    assert np.array_equal(gmm.apply(data).to_numpy(), [[0, 1], [1, 0], [0, 1], [1, 0]])
    assert np.array_equal(gmm.apply(np.array([1.0, 3.0, 0.0])), [1.0, 0.0])
    assert np.array_equal(gmm.apply(np.array([1.0, 4.0, 6.0])), [0.0, 1.0])


@pytest.mark.parametrize("D", [3, 64, 80])
@pytest.mark.parametrize("K", [1, 2, 16, 256])
def test_posteriors_match_oracle(ctx, D, K):
    rng = np.random.default_rng(D * 1000 + K)
    means, variances, w = _gmm(rng, D, K, spread=0.3)
    # rows near the components, scaled so that several components share each row's mass
    X = (means[:, rng.integers(0, K, 1000)].T + rng.standard_normal((1000, D)) * (3.0 / np.sqrt(D))).astype(np.float32)
    gmm = ks.GaussianMixtureModel(means, variances, w, ctx=ctx)
    got = gmm.apply(ctx.matrix(X)).to_numpy()
    ref = fo.gmm_posteriors(X.astype(np.float64), means, variances, w)
    # the fp64 result is stored as fp32: half an fp32 spacing of rounding on top of the 1e-12 gate
    assert (np.abs(got - ref) <= 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + 1e-12).all(), \
        np.abs(got - ref).max()
    assert np.array_equal(got == 0, ref == 0)
    assert np.allclose(got.sum(1), 1.0, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------- Fisher vectors
@pytest.mark.parametrize("D,K", [(64, 16), (80, 256), (3, 2)])
def test_fisher_vectors_match_oracle(ctx, D, K):
    rng = np.random.default_rng(D * 7 + K)
    means, variances, w = _gmm(rng, D, K, spread=0.3)
    sizes = [1, 7, 1, 300, 1000, 33, 2, 1]
    items = [(rng.standard_normal((D, n)) * 0.8).astype(np.float32) for n in sizes]
    gmm = ks.GaussianMixtureModel(means, variances, w, ctx=ctx)
    batch = ks.ItemBatch.from_items(ctx, items)
    fv = ks.FisherVector(gmm)
    out = fv.apply(batch)
    assert out.shape == (len(items), 2 * D * K)
    got = out.to_numpy(np.float32)
    for i, it in enumerate(items):
        ref = fo.matrix_vectorizer(fo.fisher_vector(it.astype(np.float64), means, variances, w))
        assert _rel(got[i].astype(np.float64), ref) <= 1e-6, (i, _rel(got[i], ref))
    again = fv.apply(batch).to_numpy(np.float32)
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32))
    single = fv.apply(items[2].astype(np.float64))
    assert single.shape == (D, 2 * K) and np.array_equal(single, got[2].reshape(2 * K, D).T)


def test_fisher_vectors_over_several_item_batches(ctx):
    """Posterior scratch of more than 256 MB splits the items into two launches of (posterior, statistics, finalize)."""
    rng = np.random.default_rng(9)
    D, K = 3, 256
    means, variances, w = _gmm(rng, D, K)
    items = [rng.standard_normal((D, n)).astype(np.float32) for n in (70000, 1, 70000)]
    gmm = ks.GaussianMixtureModel(means, variances, w, ctx=ctx)
    batch = ks.ItemBatch.from_items(ctx, items)
    l0 = ctx.launch_count()
    out = ks.FisherVector(gmm).apply(batch)
    assert ctx.launch_count() - l0 == 6
    got = out.to_numpy()
    for i, it in enumerate(items):
        ref = fo.matrix_vectorizer(fo.fisher_vector(it.astype(np.float64), means, variances, w))
        assert _rel(got[i], ref) <= 1e-6


# ---------------------------------------------------------------------------------------------------------------- row maps
def test_normalize_rows_and_signed_sqrt(ctx):
    rng = np.random.default_rng(5)
    X = (rng.standard_normal((50, 70)) * 3).astype(np.float32)
    X[3] = 0.0
    X[4] = 0.0
    X[4, 5] = 1e-30
    m = ctx.matrix(X)
    n = ks.NormalizeRows().apply(m).to_numpy()
    ref = fo.normalize_rows(X.astype(np.float64))
    assert np.abs(n - ref).max() <= 1e-7 * np.abs(ref).max()
    assert np.array_equal(n[3], np.zeros(70)) and n[4, 5] == np.float32(np.float64(np.float32(1e-30)) / 2.2e-16)
    h = ks.SignedHellingerMapper().apply(m).to_numpy(np.float32)
    assert np.array_equal(h, np.float32(fo.signed_hellinger(X.astype(np.float64))))
    assert np.array_equal(np.sign(h), np.sign(X))
    v = ks.NormalizeRows(ctx).apply(np.array([3.0, -4.0]))
    assert np.allclose(v, [0.6, -0.8])


# ---------------------------------------------------------------------------------------------------------------- rejections
def test_rejections(ctx):
    L = lib()
    img = ctx.matrix(np.zeros((2, 32 * 32 * 3), dtype=np.float32))
    out = C.c_int64(0)
    assert L.ks_lcs_extract(ctx.handle, img.handle, 32, 32, 3, 4, 6, 6, C.byref(out)) == KS_ERR_INVALID      # leaves the image
    assert L.ks_lcs_extract(ctx.handle, img.handle, 32, 31, 3, 4, 11, 6, C.byref(out)) == KS_ERR_INVALID     # shape mismatch
    assert L.ks_lcs_extract(ctx.handle, img.handle, 32, 32, 3, 4, 16, 6, C.byref(out)) == KS_ERR_INVALID     # no keypoint
    assert L.ks_lcs_extract(ctx.handle, img.handle, 32, 32, 3, 0, 11, 6, C.byref(out)) == KS_ERR_INVALID     # stride 0
    assert L.ks_lcs_extract(ctx.handle, img.handle, 32, 32, 3, 4, 11, 6, C.byref(out)) == 0
    rng = np.random.default_rng(6)
    means, variances, w = _gmm(rng, 4, 3)

    def create(mu=means, var=variances, wt=w, thr=1e-4, dim=4, k=3):
        mu, var, wt = (np.asfortranarray(a, dtype=np.float64) for a in (mu, var, wt))
        return L.ks_gmm_create(ctx.handle, mu.ctypes.data_as(C.c_void_p), var.ctypes.data_as(C.c_void_p), wt.ctypes.data_as(C.c_void_p),
                               dim, k, thr, C.byref(out))

    bad_mu = means.copy()
    bad_mu[1, 2] = np.nan
    for kw in ({"mu": bad_mu}, {"var": np.where(np.arange(12).reshape(4, 3) == 5, 0.0, variances)},
               {"var": np.where(np.arange(12).reshape(4, 3) == 5, -1.0, variances)}, {"var": variances * np.inf},
               {"wt": np.array([0.5, 0.5, 0.0])}, {"wt": np.array([0.5, np.nan, 0.5])}, {"thr": 1.0 / 3}, {"thr": -1e-9},
               {"thr": np.nan}, {"dim": 0}, {"k": 0}):
        assert create(**kw) == KS_ERR_INVALID, kw
    with pytest.raises(ks.KeystoneError):
        ks.GaussianMixtureModel(means, variances, w, weightThreshold=0.5, ctx=ctx)
    assert create() == 0
    g = out.value
    x5 = ctx.matrix(np.zeros((10, 5), dtype=np.float32))
    x4 = ctx.matrix(np.zeros((10, 4), dtype=np.float32))
    assert L.ks_gmm_posteriors(ctx.handle, g, x5.handle, C.byref(out)) == KS_ERR_INVALID                  # cols != D
    assert L.ks_gmm_posteriors(ctx.handle, 987654, x4.handle, C.byref(out)) == KS_ERR_HANDLE

    def fv(offs, x=x4, n=None):
        o = np.ascontiguousarray(offs, dtype=np.int64)
        return L.ks_fisher_vector_apply(ctx.handle, g, x.handle, o.ctypes.data_as(C.c_void_p), len(o) - 1 if n is None else n,
                                        C.byref(out))

    assert fv([0, 6, 4, 10]) == KS_ERR_INVALID     # not monotone
    assert fv([0, 4, 9]) == KS_ERR_INVALID         # last offset != rows
    assert fv([0, 4, 4, 10]) == KS_ERR_INVALID     # empty item
    assert fv([1, 4, 10]) == KS_ERR_INVALID        # first offset != 0
    assert fv([0, 10], x=x5) == KS_ERR_INVALID     # cols != D
    assert fv([0], n=0) == KS_ERR_INVALID          # no item
    assert fv([0, 3, 10]) == 0
    assert L.ks_gmm_destroy(ctx.handle, g) == 0
    assert L.ks_gmm_destroy(ctx.handle, g) == KS_ERR_HANDLE
    assert L.ks_matrix_map(ctx.handle, x4.handle, 3, None, 0.0, 0.0, C.byref(out)) == KS_ERR_INVALID
    with pytest.raises(ValueError):
        ks.ItemBatch(x4, [0, 5, 4, 10])


# ---------------------------------------------------------------------------------------------------------------- end to end
def test_miniature_lcs_branch_into_bwls(ctx):
    """LCSExtractor -> BatchPCATransformer (device path) -> FisherVector -> FloatToDouble -> MatrixVectorizer -> NormalizeRows ->
    SignedHellingerMapper -> NormalizeRows on synthetic images, against the oracle fed the device's PCA output; then the C5 solver
    (BlockWeightedLeastSquaresEstimator, mixture weight 0.25) on those features with random labels, within the BWLS gate."""
    rng = np.random.default_rng(7)
    n, k = 240, 4
    imgs = (rng.random((n, 32, 32, 3)) * 255).astype(np.float32)
    lcs = ks.LCSExtractor(4, 8, 4).apply(ks.ImageBatch.from_images(ctx, imgs))
    desc = lcs.matrix.to_numpy()
    pca_mat = po.compute_pca(desc, 8)
    z = ks.BatchPCATransformer(ks.PCATransformer.from_matrix(ctx, pca_mat)).apply(lcs)
    assert isinstance(z, ks.ItemBatch) and np.array_equal(z.offsets, lcs.offsets)
    zl = z.to_list()
    allz = np.concatenate(zl, 1)
    means = allz[:, rng.choice(allz.shape[1], 4, replace=False)]
    variances = np.repeat(allz.var(1)[:, None], 4, 1)
    gmm = ks.GaussianMixtureModel(means, variances, np.full(4, 0.25), ctx=ctx)
    feats = ks.Pipeline([ks.FisherVector(gmm), ks.FloatToDouble(), ks.MatrixVectorizer(), ks.NormalizeRows(), ks.SignedHellingerMapper(),
                         ks.NormalizeRows()])(z)
    F = feats.to_numpy()
    ref = fo.fv_tail(zl, means, variances, np.full(4, 0.25))
    assert F.shape == (n, 64)
    for i in range(n):
        assert _rel(F[i], ref[i]) <= 1e-5, (i, _rel(F[i], ref[i]))
    cls = rng.integers(0, k, n)
    Y = ko.class_label_indicators(cls, k)
    lam, w = 6e-5, 0.25   # the C5 setting (ImageNetSiftLcsFV.scala)
    assert bo.cond_bound(F, Y, 32, lam, w) <= 1e3
    model = ks.BlockWeightedLeastSquaresEstimator(32, 2, lam, w).fit(feats, ctx.labels_from_classes(cls, k))
    xs, _ = ko.bwls_fit(F, Y, 32, 2, lam, w)
    assert _rel(np.concatenate(model.xs, 0), np.concatenate(xs, 0)) <= W_TOL
