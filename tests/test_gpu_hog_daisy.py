"""HogExtractor and DaisyExtractor on the H100 against the reference suites' MATLAB sums on images/gantrycrane.png and against the
NumPy restatement (tests/hog_daisy_oracle.py) fed the same inputs.

Gate (device against oracle): >= 99.9 % of entries bit-identical, none more than 1 fp32 ulp apart, and for DAISY the same zeroed
histograms.  The kernels take every rounding step the oracle takes, in the same order, so the expected result is bit identity."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import KeystoneError, check, lib
from oracle import keystone_oracle as ko

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fv_oracle as fo  # noqa: E402
import gmm_oracle as go  # noqa: E402
import hog_daisy_oracle as hd  # noqa: E402
import sift_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu
KS_ERR_INVALID = -1


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def bgr(golden_dir):
    """images/gantrycrane.png as ImageUtils.loadImage yields it: (x = row, y, c) with c in BGR order."""
    return np.load(os.path.join(golden_dir, "conv_gantrycrane.npz"))["rgb"][:, :, ::-1].astype(np.float32)


def _ulps(a, b):
    return np.abs(np.asarray(a, np.float32).view(np.int32).astype(np.int64) - np.asarray(b, np.float32).view(np.int32).astype(np.int64))


def _gate(dev, ref, daisy_h=None):
    assert dev.shape == ref.shape, (dev.shape, ref.shape)
    if dev.size == 0:
        return
    u = _ulps(dev, ref)
    assert u.max() <= 1, u.max()
    assert (u == 0).mean() >= 0.999, (u == 0).mean()
    if daisy_h:
        zd = (dev.reshape(dev.shape[0], -1, daisy_h) == 0).all(2)
        zo = (ref.reshape(ref.shape[0], -1, daisy_h) == 0).all(2)
        assert np.array_equal(zd, zo)


def _gray_batch(ctx, grays):
    return ks.ImageBatch.from_images(ctx, np.stack(grays)[..., None].astype(np.float32))


# ------------------------------------------------------------------------------------------------------------------------ HOG
def test_hog_gantrycrane_matches_matlab_and_oracle(ctx, bgr):
    """HogExtractorSuite through PixelScaler -> HogExtractor(50 | 8): the fp32 column-major sums within 1e-8 and 1e-4 of MATLAB."""
    batch = ks.ImageBatch.from_images(ctx, bgr[None])
    scaled = ks.PixelScaler().apply(batch)
    for bin_, matlab, tol in ((50, 59.2162514, 1e-8), (8, 4.5775269e+03, 1e-4)):
        items = ks.HogExtractor(bin_).apply(scaled)
        assert isinstance(items, ks.ItemBatch) and items.cols == 32
        F = items.to_numpy(np.float32)
        assert items.offsets.tolist() == [0, hd.hog_rows(264, 400, bin_)]
        ours = hd.breeze_sum_f32(F)
        assert abs((ours - matlab) / ours) < tol, (bin_, (ours - matlab) / ours)
        _gate(F, hd.hog_extract(bgr.astype(np.float64) / 255.0, bin_))
    # one image in: the reference's (cells x 32) matrix, unscaled values when no PixelScaler precedes
    single = ks.HogExtractor(8, ctx=ctx).apply(bgr)
    _gate(single, hd.hog_extract(bgr.astype(np.float64), 8))


# odd shapes: bins that do not divide the image, rows that wrap into the next column, fewer than 3 cells, a single cell row
HOG_CASES = [((23, 17), 4), ((21, 31), 6), ((25, 26), 5), ((17, 12), 3), ((40, 31), 7), ((9, 40), 4), ((30, 30), 10),
             ((64, 48), 8), ((2, 2), 1), ((61, 44), 2)]


@pytest.mark.parametrize("shape,bin_", HOG_CASES)
def test_hog_synthetic_device_against_oracle(ctx, shape, bin_):
    rng = np.random.default_rng(shape[0] * 1000 + shape[1] * 10 + bin_)
    imgs = rng.integers(0, 256, size=(3,) + shape + (3,)).astype(np.float32)
    imgs[1, :, :, 1] = imgs[1, :, :, 2]           # ties in the channel scan
    imgs[2, : shape[0] // 2] = 128.0              # a flat region: zero gradients and zero histograms
    items = ks.HogExtractor(bin_).apply(ks.PixelScaler().apply(ks.ImageBatch.from_images(ctx, imgs)))
    rows = hd.hog_rows(*shape, bin_)
    assert items.offsets.tolist() == [0, rows, 2 * rows, 3 * rows]
    F = items.to_numpy(np.float32)
    for i in range(3):
        _gate(F[i * rows:(i + 1) * rows], hd.hog_extract(imgs[i].astype(np.float64) / 255.0, bin_))


# ---------------------------------------------------------------------------------------------------------------------- DAISY
def test_daisy_gantrycrane_matches_matlab_and_oracle(ctx, bgr):
    """DaisyExtractorSuite through GrayScaler -> DaisyExtractor(): first keypoint within 1e-5 and the full sum within 1e-7 of
    MATLAB; (200 x nKP) per image like SIFT's (128 x nKP)."""
    gray = ks.GrayScaler().apply(ks.ImageBatch.from_images(ctx, bgr[None]))
    de = ks.DaisyExtractor()
    items = de.apply(gray)
    assert items.offsets.tolist() == [0, 5336] and items.cols == de.daisyFeatureSize == 200
    D = items.to_list(np.float64)[0]
    assert D.shape == (200, 5336)
    first, total = 55.127217737738533, 3.240635661296463E5
    assert abs((D[:, 0].sum() - first) / first) < 1e-5
    assert abs((D.sum() - total) / total) < 1e-7
    g32 = gray.matrix.to_numpy(np.float32)[0].reshape(400, 264).T
    _gate(items.to_numpy(np.float32), hd.daisy_extract(g32.astype(np.float64)), 8)
    assert ks.SIFTExtractor(scaleStep=2).apply(gray).to_list()[0].shape[0] == 128   # same orientation as SIFT


# (shape, (T, Q, R, H, border, stride)): defaults, no keypoint, one keypoint, flat images (zeroed histograms), odd settings
DAISY_CASES = [((48, 40), (8, 3, 7, 8, 16, 4)), ((33, 33), (8, 3, 7, 8, 16, 4)), ((20, 20), (8, 3, 7, 8, 16, 4)),
               ((37, 41), (5, 2, 6, 4, 7, 9)), ((50, 29), (4, 1, 3, 3, 3, 5)), ((45, 52), (12, 4, 9, 6, 10, 3)),
               ((31, 27), (3, 2, 2, 2, 2, 1)), ((26, 35), (8, 3, 7, 1, 9, 6))]


@pytest.mark.parametrize("shape,params", DAISY_CASES)
def test_daisy_synthetic_device_against_oracle(ctx, shape, params):
    rng = np.random.default_rng(hash((shape, params)) % 2**32)
    x, y = np.meshgrid(np.arange(shape[0]), np.arange(shape[1]), indexing="ij")
    grays = [(100 + 60 * np.sin(x / (2.0 + k)) * np.cos(y / 4.0) + 10 * rng.standard_normal(shape)).astype(np.float32) for k in range(2)]
    grays.append(np.zeros(shape, dtype=np.float32))            # no gradient anywhere: every histogram zeroed
    de = ks.DaisyExtractor(*params)
    items = de.apply(_gray_batch(ctx, grays))
    nkp = de.keypoints(*shape)
    assert items.offsets.tolist() == [0, nkp, 2 * nkp, 3 * nkp] and items.cols == de.daisyFeatureSize
    D = items.to_numpy(np.float32)
    for i, g in enumerate(grays):
        _gate(D[i * nkp:(i + 1) * nkp], hd.daisy_extract(g.astype(np.float64), *params), params[3])
    if nkp:
        assert not D[2 * nkp:].any()


# ------------------------------------------------------------------------------------------------------------------- both nodes
def test_repeatable_and_mixed_shapes_keep_order(ctx):
    rng = np.random.default_rng(8)
    rgbs = [rng.integers(0, 256, size=s).astype(np.float32) for s in ((41, 37, 3), (52, 44, 3), (41, 37, 3), (36, 36, 3))]
    hog = ks.HogExtractor(6, ctx=ctx)
    got = hog.apply(ks.PixelScaler(ctx=ctx).apply(rgbs))      # a list of one-image scaled batches
    assert isinstance(got, ks.ItemBatch) and got.n_items == 4
    host = got.to_numpy(np.float32)
    for k, im in enumerate(rgbs):
        assert got.offsets[k + 1] - got.offsets[k] == hog.cells(*im.shape[:2])
        _gate(host[got.offsets[k]:got.offsets[k + 1]], hd.hog_extract(im.astype(np.float64) / 255.0, 6))
    plain = hog.apply(rgbs)                                    # a list of arrays: grouped by shape, input order kept
    for k, im in enumerate(rgbs):
        _gate(plain.to_numpy(np.float32)[plain.offsets[k]:plain.offsets[k + 1]], hd.hog_extract(im.astype(np.float64), 6))
    b = ks.ImageBatch.from_images(ctx, np.stack([rgbs[0], rgbs[2]] * 4))
    assert np.array_equal(hog.apply(b).to_numpy(np.float32), hog.apply(b).to_numpy(np.float32))

    grays = [rng.random(s).astype(np.float32) * 255 for s in ((50, 44), (61, 40), (50, 44), (45, 45))]
    de = ks.DaisyExtractor(ctx=ctx)
    items = de.apply([g[:, :, None] for g in grays])
    assert items.n_items == 4
    for g, item in zip(grays, items.to_list(np.float32)):
        assert item.shape == (200, de.keypoints(*g.shape))
        _gate(item.T.copy(), hd.daisy_extract(g.astype(np.float64)), 8)
    assert np.array_equal(de.apply(grays[1]), items.to_list(np.float32)[1])
    gb = _gray_batch(ctx, [grays[0], grays[2]] * 4)
    assert np.array_equal(de.apply(gb).to_numpy(np.float32), de.apply(gb).to_numpy(np.float32))


def test_rejections(ctx):
    rng = np.random.default_rng(9)
    h = C.c_int64(0)

    def rejected(rc_call, text=None):
        with pytest.raises(KeystoneError) as ei:
            check(ctx.handle, rc_call())
        assert ei.value.code == KS_ERR_INVALID
        if text:
            assert text in str(ei.value)

    rgb = ks.ImageBatch.from_images(ctx, rng.random((1, 30, 30, 3)).astype(np.float32) * 255)
    m = rgb.matrix.handle
    rejected(lambda: lib().ks_hog_extract(ctx.handle, m, 30, 30, 3, 1, 0, C.byref(h)))        # bin < 1
    rejected(lambda: lib().ks_hog_extract(ctx.handle, m, 30, 30, 3, 1, 1025, C.byref(h)))     # bin too large
    rejected(lambda: lib().ks_hog_extract(ctx.handle, m, 30, 29, 3, 1, 4, C.byref(h)))        # shape does not match
    rejected(lambda: lib().ks_hog_extract(ctx.handle, m, 0, 30, 3, 1, 4, C.byref(h)))
    rejected(lambda: lib().ks_hog_extract(ctx.handle, m, 30, 30, 3, 2, 4, C.byref(h)))        # pixel_scale
    rejected(lambda: lib().ks_hog_extract(ctx.handle, m, 45, 30, 2, 1, 4, C.byref(h)))        # two channels
    one = _gray_batch(ctx, [rng.random((30, 30)).astype(np.float32)])
    with pytest.raises(KeystoneError) as ei:
        ks.HogExtractor(4).apply(one)                                                           # one channel
    assert ei.value.code == KS_ERR_INVALID
    # 23 x 23 at bin 4: both sides round up to 24 and the reference's last read passes the end of the image
    wrap = ks.ImageBatch.from_images(ctx, rng.random((1, 23, 23, 3)).astype(np.float32))
    with pytest.raises(KeystoneError) as ei:
        ks.HogExtractor(4).apply(wrap)
    assert ei.value.code == KS_ERR_INVALID and "past the end" in str(ei.value)

    g = _gray_batch(ctx, [rng.random((48, 48)).astype(np.float32)])
    gm = g.matrix.handle
    for T, Q, R, H, border, stride in ((0, 3, 7, 8, 16, 4), (8, 0, 7, 8, 16, 4), (8, 3, 0, 8, 16, 4), (8, 3, 7, 0, 16, 4),
                                       (8, 3, 7, 8, -1, 4), (8, 3, 7, 8, 16, 0), (65, 3, 7, 8, 16, 4), (8, 17, 7, 8, 16, 4),
                                       (8, 3, 7, 65, 16, 4), (8, 1, 4000, 8, 16, 4)):
        rejected(lambda: lib().ks_daisy_extract(ctx.handle, gm, 48, 48, T, Q, R, H, border, stride, C.byref(h)))
    rejected(lambda: lib().ks_daisy_extract(ctx.handle, gm, 48, 47, 8, 3, 7, 8, 16, 4, C.byref(h)))    # shape
    rejected(lambda: lib().ks_daisy_extract(ctx.handle, gm, 48, 48, 8, 3, 7, 8, 6, 4, C.byref(h)), "leaves the image")
    rejected(lambda: lib().ks_daisy_extract(ctx.handle, rgb.matrix.handle, 30, 30, 8, 3, 7, 8, 8, 4, C.byref(h)))  # 3 channels
    bad = rng.random((48, 48)).astype(np.float32)
    bad[5, 6] = np.nan
    with pytest.raises(KeystoneError) as ei:
        ks.DaisyExtractor().apply(_gray_batch(ctx, [bad]))
    assert ei.value.code == KS_ERR_INVALID and "non-finite" in str(ei.value)
    inf = rng.random((1, 30, 30, 3)).astype(np.float32)
    inf[0, 2, 3, 1] = np.inf
    with pytest.raises(KeystoneError) as ei:
        ks.HogExtractor(5).apply(ks.PixelScaler().apply(ks.ImageBatch.from_images(ctx, inf)))
    assert ei.value.code == KS_ERR_INVALID and "non-finite" in str(ei.value)
    # no keypoint / no interior cell: an empty item batch
    assert ks.DaisyExtractor().apply(_gray_batch(ctx, [rng.random((20, 20)).astype(np.float32)])).offsets.tolist() == [0, 0]
    assert ks.HogExtractor(4).apply(ks.ImageBatch.from_images(ctx, np.ones((2, 9, 40, 3), np.float32))).offsets.tolist() == [0, 0, 0]


def _rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(np.asarray(a) - b) / max(np.linalg.norm(b), 1e-300))


def test_miniature_voc_branch_with_daisy(ctx):
    """PixelScaler -> GrayScaler -> DaisyExtractor -> ColumnSampler -> ColumnPCAEstimator(80) -> GMMFisherVectorEstimator(16) ->
    FloatToDouble -> MatrixVectorizer -> NormalizeRows -> SignedHellingerMapper -> NormalizeRows -> BlockLeastSquaresEstimator:
    VOCSIFTFisher with DAISY in SIFT's place, each stage against the oracles fed the device's previous stage, within the gates of
    tests/test_gpu_sift.py."""
    rng = np.random.default_rng(12)
    n, k = 24, 3
    x, y = np.meshgrid(np.arange(56), np.arange(48), indexing="ij")
    rgbs = []
    for i in range(n):
        base = 128 + 100 * np.sin(x / (2.0 + i % 5) + i) * np.cos(y / (3.0 + i % 3))
        rgbs.append(np.clip(base[..., None] + 20 * rng.standard_normal((56, 48, 3)), 0, 255).astype(np.uint8))
    batch = ks.ImageBatch.from_images(ctx, np.stack([r[:, :, ::-1] for r in rgbs]).astype(np.float32))
    daisy = ks.DaisyExtractor().apply(ks.GrayScaler().apply(ks.PixelScaler().apply(batch)))
    desc = daisy.to_numpy(np.float32)
    nkp = daisy.offsets[1]
    assert nkp == 6 * 4
    for i in (0, n - 1):
        _gate(desc[i * nkp:(i + 1) * nkp], hd.daisy_extract(so.gray_f32(rgbs[i]).astype(np.float64)), 8)
    sample = ks.ColumnSampler(200, seed=2).apply(daisy)
    pca = ks.ColumnPCAEstimator(80, ctx=ctx).fit(sample.to_list(np.float32))
    zs = pca.apply(sample)
    est = ks.GMMFisherVectorEstimator(16, ctx=ctx)
    fv = est.fit(zs)
    ref = go.gmm_fit(zs.matrix.to_numpy(), 16, uniforms=est.gmm_estimator.uniforms(80))
    assert est.gmm_estimator.stats["iterations"] == ref["iterations"]
    assert _rel(fv.gmm.means, ref["means"]) <= 1e-9 and _rel(fv.gmm.variances, ref["variances"]) <= 1e-9
    z = pca.apply(daisy)
    feats = ks.Pipeline([fv, ks.FloatToDouble(), ks.MatrixVectorizer(), ks.NormalizeRows(), ks.SignedHellingerMapper(),
                         ks.NormalizeRows()])(z)
    F = feats.to_numpy()
    tail = fo.fv_tail(z.to_list(), ref["means"], ref["variances"], ref["weights"])
    assert F.shape == (n, 2 * 80 * 16)
    for i in range(n):
        assert _rel(F[i], tail[i]) <= 1e-5, (i, _rel(F[i], tail[i]))
    cls = rng.integers(0, k, n)
    model = ks.BlockLeastSquaresEstimator(640, 1, 1.0).fit(feats, ctx.labels_from_classes(cls, k))
    xs, _, _ = ko.block_ls_fit(F, ko.class_label_indicators(cls, k), 640, 1, 1.0)
    assert _rel(np.concatenate(model.xs, 0), np.concatenate(xs, 0)) <= 5e-5
