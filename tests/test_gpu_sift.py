"""PixelScaler, GrayScaler and SIFTExtractor on the H100 against the NumPy restatement (tests/sift_oracle.py) fed the same fp32 gray
images, and against the reference's own descriptors of images/000012.jpg (feats128.csv: the fixture keeps the zero / nonzero
status of all 64 990 keypoints and the full descriptors of every 32nd).

Gates (device against oracle): identical keypoint counts and order; identical zero masks except keypoints whose oracle mass lies
within 1e-5 relative of the 0.005 threshold; >= 99.9 % of entries bit-identical and none off by more than 1.  Device against
feats128: the oracle's own gate (>= 99.5 % same zero status over all keypoints, and over the sampled ones >= 99 % within 1 and
>= 95 % exact where both are nonzero)."""
import os
import sys

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import KeystoneError
from oracle import keystone_oracle as ko

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fv_oracle as fo  # noqa: E402
import gmm_oracle as go  # noqa: E402
import sift_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu
KS_ERR_INVALID = -1


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "sift_000012.npz"))
    return z["rgb"], z["zero"], z["cols"], z["feats"]


def _bgr_batch(rgbs):
    """8-bit RGB files as ImageUtils.loadImage yields them: (n, x, y, c) with c in BGR order."""
    return np.stack([np.asarray(r)[:, :, ::-1] for r in rgbs]).astype(np.float32)


def _gray_batch(ctx, grays):
    return ks.ImageBatch.from_images(ctx, np.stack(grays)[..., None])


def _check_against_oracle(dev, gray, params):
    D, mass = so.sift_extract(gray, *params, with_mass=True)
    assert dev.shape == D.shape, (dev.shape, D.shape)
    zd, zo = (dev == 0).all(1), (D == 0).all(1)
    near = np.abs(mass.astype(np.float64) - 0.005) <= 1e-5 * 0.005
    assert np.array_equal(zd[~near], zo[~near])
    keep = ~near
    diff = np.abs(dev[keep] - D[keep])
    assert diff.size == 0 or diff.max() <= 1
    assert diff.size == 0 or (diff == 0).mean() >= 0.999, (diff == 0).mean()
    return D


def test_gray_and_pixel_scaler_bit_identical(ctx):
    rng = np.random.default_rng(3)
    rgbs = [rng.integers(0, 256, size=(37, 23, 3), dtype=np.uint8) for _ in range(3)]
    batch = ks.ImageBatch.from_images(ctx, _bgr_batch(rgbs))
    gray = ks.GrayScaler().apply(ks.PixelScaler().apply(batch))
    assert (gray.x_dim, gray.y_dim, gray.channels) == (37, 23, 1)
    got = gray.matrix.to_numpy(np.float32)
    for i, r in enumerate(rgbs):
        assert np.array_equal(got[i], ks.images_to_matrix(so.gray_f32(r)[None, :, :, None])[0])
    scaled = ks.PixelScaler().apply(batch).matrix.to_numpy(np.float32)
    assert np.array_equal(scaled, (batch.matrix.to_numpy(np.float64) / 255.0).astype(np.float32))
    # GrayScaler alone on unscaled values, and on one channel (sqrt of the mean square = |v|)
    g2 = ks.GrayScaler().apply(batch).matrix.to_numpy(np.float32)
    assert np.array_equal(g2[0], ks.images_to_matrix(so.gray_scale(_bgr_batch(rgbs[:1])[0]).astype(np.float32)[None, :, :, None])[0])
    one = ks.ImageBatch.from_images(ctx, -np.abs(rng.standard_normal((2, 5, 4, 1))).astype(np.float32))
    assert np.array_equal(ks.GrayScaler().apply(one).matrix.to_numpy(np.float32), np.abs(one.matrix.to_numpy(np.float32)))


def test_fixture_device_against_oracle_and_feats128(ctx, fixture):
    rgb, zero, cols, feats = fixture
    batch = ks.ImageBatch.from_images(ctx, _bgr_batch([rgb]))
    gray_dev = ks.GrayScaler().apply(ks.PixelScaler().apply(batch))
    gray = so.gray_f32(rgb)
    assert np.array_equal(gray_dev.matrix.to_numpy(np.float32)[0], ks.images_to_matrix(gray[None, :, :, None])[0])
    items = ks.SIFTExtractor(scaleStep=0).apply(gray_dev)
    assert isinstance(items, ks.ItemBatch) and items.cols == 128 and items.offsets.tolist() == [0, 64990]
    dev = items.matrix.to_numpy(np.float32)
    _check_against_oracle(dev, gray, (3, 4, 4, 0))
    zd = (dev == 0).all(1)
    assert (zero == zd).mean() >= 0.995
    ref, ds = feats.T.astype(np.float32), dev[cols]
    both = ~zero[cols] & ~zd[cols]
    diff = np.abs(ds[both] - ref[both])
    assert (diff <= 1).mean() >= 0.99 and (diff == 0).mean() >= 0.95
    # the reference's layout: one (128 x nKP) matrix per image
    assert np.array_equal(items.to_list(np.float32)[0], dev.T)


# shapes where a scale has no frames (30 x 30 at the defaults: 9, 4, 1, 0) or exactly one, odd shapes, and parameter variants
CASES = [((30, 30), (3, 4, 4, 1)), ((29, 31), (3, 4, 4, 0)), ((61, 47), (3, 4, 4, 1)), ((75, 50), (3, 4, 4, 0)),
         ((53, 88), (2, 3, 3, 2)), ((41, 40), (5, 6, 2, 0)), ((13, 13), (1, 4, 1, 0)), ((70, 66), (3, 4, 5, 1)),
         ((12, 9), (3, 4, 4, 1))]


@pytest.mark.parametrize("shape,params", CASES)
def test_synthetic_device_against_oracle(ctx, shape, params):
    rng = np.random.default_rng(hash((shape, params)) % 2**32)
    # smooth structure plus noise, so that both thresholded and textured keypoints occur
    x, y = np.meshgrid(np.arange(shape[0]), np.arange(shape[1]), indexing="ij")
    grays = []
    for k in range(3):
        g = 0.5 + 0.3 * np.sin(x / (3.0 + k)) * np.cos(y / 5.0) + 0.05 * rng.standard_normal(shape)
        g[: shape[0] // 3] *= 0.02   # a nearly flat band: keypoints below the contrast threshold
        grays.append(g.astype(np.float32))
    se = ks.SIFTExtractor(*params)
    nkp = se.keypoints(*shape)
    assert se.keypoints_per_scale(*shape) == so.keypoint_counts(*shape, *params)
    items = se.apply(_gray_batch(ctx, grays))
    assert items.offsets.tolist() == [0, nkp, 2 * nkp, 3 * nkp]
    dev = items.matrix.to_numpy(np.float32)
    for i, g in enumerate(grays):
        _check_against_oracle(dev[i * nkp:(i + 1) * nkp], g, params)


def test_repeatable_and_mixed_shapes_keep_order(ctx):
    rng = np.random.default_rng(5)
    ims = [rng.random(s).astype(np.float32) for s in ((40, 33), (52, 40), (40, 33), (35, 35))]
    se = ks.SIFTExtractor(ctx=ctx)
    got = se.apply([im[:, :, None] for im in ims])
    assert isinstance(got, ks.ItemBatch) and got.n_items == 4
    for im, item in zip(ims, got.to_list(np.float32)):
        assert item.shape == (128, se.keypoints(*im.shape))
        _check_against_oracle(item.T.copy(), im, (3, 4, 4, 1))
    b = _gray_batch(ctx, [ims[0], ims[2]] * 5)
    a1 = se.apply(b).matrix.to_numpy(np.float32)
    a2 = se.apply(b).matrix.to_numpy(np.float32)
    assert np.array_equal(a1, a2)
    single = se.apply(ims[1])
    assert np.array_equal(single, got.to_list(np.float32)[1])
    # a list of RGB images through the whole head: one batch per image, input order kept
    rgbs = [rng.integers(0, 256, size=s, dtype=np.uint8) for s in ((36, 31, 3), (44, 30, 3), (36, 31, 3))]
    grays = ks.GrayScaler().apply(ks.PixelScaler(ctx=ctx).apply([r[:, :, ::-1].astype(np.float32) for r in rgbs]))
    chain = ks.SIFTExtractor().apply(grays)
    assert chain.n_items == 3
    for r, item in zip(rgbs, chain.to_list(np.float32)):
        _check_against_oracle(item.T.copy(), so.gray_f32(r), (3, 4, 4, 1))


def test_rejections(ctx):
    rng = np.random.default_rng(6)
    g = _gray_batch(ctx, [rng.random((30, 30)).astype(np.float32)])
    for params in ((0, 4, 4, 1), (3, 0, 4, 1), (3, 4, 0, 1), (3, 4, 4, -1)):
        with pytest.raises(KeystoneError) as ei:
            ks.SIFTExtractor(*params).apply(g)
        assert ei.value.code == KS_ERR_INVALID
    rgb = ks.ImageBatch.from_images(ctx, rng.random((1, 30, 30, 3)).astype(np.float32))
    with pytest.raises(KeystoneError):
        ks.SIFTExtractor().apply(rgb)                     # three channels
    from keystone_b200._capi import check, lib
    import ctypes as C
    h = C.c_int64(0)
    with pytest.raises(KeystoneError) as ei:              # shape does not match the matrix
        check(ctx.handle, lib().ks_sift_extract(ctx.handle, g.matrix.handle, 30, 29, 3, 4, 4, 1, C.byref(h)))
    assert ei.value.code == KS_ERR_INVALID
    with pytest.raises(KeystoneError) as ei:
        check(ctx.handle, lib().ks_image_grayscale(ctx.handle, rgb.matrix.handle, 30, 30, 2, 1, C.byref(h)))
    assert ei.value.code == KS_ERR_INVALID
    with pytest.raises(KeystoneError) as ei:
        check(ctx.handle, lib().ks_image_grayscale(ctx.handle, rgb.matrix.handle, 30, 30, 3, 2, C.byref(h)))
    assert ei.value.code == KS_ERR_INVALID
    bad = rng.random((30, 30)).astype(np.float32)
    bad[3, 4] = np.nan
    for node, data in ((ks.SIFTExtractor(), _gray_batch(ctx, [bad])), (ks.GrayScaler(), _gray_batch(ctx, [bad]))):
        with pytest.raises(KeystoneError) as ei:
            node.apply(data)
        assert ei.value.code == KS_ERR_INVALID and "non-finite" in str(ei.value)
    inf = rng.random((1, 30, 30, 3)).astype(np.float32)
    inf[0, 1, 1, 2] = np.inf
    with pytest.raises(KeystoneError):
        ks.PixelScaler().apply(ks.ImageBatch.from_images(ctx, inf)).matrix
    # a scale-free shape: every scale without frames gives an empty item batch
    tiny = ks.SIFTExtractor().apply(_gray_batch(ctx, [rng.random((8, 8)).astype(np.float32)]))
    assert tiny.rows == 0 and tiny.offsets.tolist() == [0, 0]


def _rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(np.asarray(a) - b) / max(np.linalg.norm(b), 1e-300))


def test_miniature_voc_branch(ctx):
    """PixelScaler -> GrayScaler -> SIFTExtractor -> ColumnSampler -> ColumnPCAEstimator(80) -> GMMFisherVectorEstimator(16) ->
    FloatToDouble -> MatrixVectorizer -> NormalizeRows -> SignedHellingerMapper -> NormalizeRows -> BlockLeastSquaresEstimator on
    synthetic images (VOCSIFTFisher.scala), each stage against the oracles fed the device's previous stage, within the gates of
    tests/test_gpu_gmm.py (EM 1e-9, Fisher vectors 1e-5 per image) and the parity-mode block solver (5e-5)."""
    rng = np.random.default_rng(11)
    n, k = 24, 3
    x, y = np.meshgrid(np.arange(48), np.arange(40), indexing="ij")
    rgbs = []
    for i in range(n):
        base = 128 + 100 * np.sin(x / (2.0 + i % 5) + i) * np.cos(y / (3.0 + i % 3))
        rgbs.append(np.clip(base[..., None] + 20 * rng.standard_normal((48, 40, 3)), 0, 255).astype(np.uint8))
    batch = ks.ImageBatch.from_images(ctx, _bgr_batch(rgbs))
    sift = ks.SIFTExtractor(3, 4, 4, 0).apply(ks.GrayScaler().apply(ks.PixelScaler().apply(batch)))
    desc = sift.matrix.to_numpy(np.float32)
    nkp = sift.offsets[1]
    for i in (0, n - 1):
        _check_against_oracle(desc[i * nkp:(i + 1) * nkp], so.gray_f32(rgbs[i]), (3, 4, 4, 0))
    sample = ks.ColumnSampler(200, seed=2).apply(sift)
    pca = ks.ColumnPCAEstimator(80, ctx=ctx).fit(sample.to_list(np.float32))
    zs = pca.apply(sample)
    est = ks.GMMFisherVectorEstimator(16, ctx=ctx)
    fv = est.fit(zs)
    ref = go.gmm_fit(zs.matrix.to_numpy(), 16, uniforms=est.gmm_estimator.uniforms(80))
    assert est.gmm_estimator.stats["iterations"] == ref["iterations"]
    assert _rel(fv.gmm.means, ref["means"]) <= 1e-9 and _rel(fv.gmm.variances, ref["variances"]) <= 1e-9
    z = pca.apply(sift)
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
