"""The CIFAR random-patch front end and test-time augmentation on the H100 against tests/augment_oracle.py and the existing oracles:
image views (bit-identical), the Convolver over views (against the Convolver over the materialised views), Stats.normalizeRows
(<= 1 fp32 ulp), StandardScaler (1e-12 relative, <= 1 ulp, bit-identical refit), the grouped evaluator (exact counts), every
rejection, and both pipelines end to end in miniature."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import keystone_b200 as ks
from keystone_b200 import pipelines
from keystone_b200._capi import lib
from oracle import keystone_oracle as ko

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import augment_oracle as ao  # noqa: E402

pytestmark = pytest.mark.gpu
KS_ERR_INVALID = -1


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def img000012(golden_dir):
    return np.load(os.path.join(golden_dir, "sift_000012.npz"))["rgb"].astype(np.float32)


def _ulps(a, b):
    return np.abs(np.asarray(a, np.float32).view(np.int32).astype(np.int64) - np.asarray(b, np.float32).view(np.int32).astype(np.int64))


def _oracle_views(images, views, px, py):
    return np.stack([ao.vectorize(ao.flip_horizontal(ao.crop(images[i], sx, sy, sx + px, sy + py)) if f else
                                  ao.crop(images[i], sx, sy, sx + px, sy + py)) for i, sx, sy, f in views]).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------ image views
def test_image_views_bit_identical_with_border_and_flips(ctx):
    rng = np.random.default_rng(1)
    imgs = rng.standard_normal((5, 20, 17, 3)).astype(np.float32)
    batch = ks.ImageBatch.from_images(ctx, imgs)
    views = [(0, 0, 0, 0), (4, 13, 9, 1), (2, 0, 9, 1), (3, 13, 0, 0), (1, 6, 4, 1), (4, 13, 9, 0)]
    got = ks.ImageViews(batch, views, 7, 8).to_numpy(np.float32)
    assert np.array_equal(got, _oracle_views(imgs, views, 7, 8))


def test_patchers_on_real_image_bit_identical(ctx, img000012):
    batch = ks.ImageBatch.from_images(ctx, img000012[None])
    px, py = img000012.shape[0] // 2, img000012.shape[1] // 2
    wins = ks.Windower(100, 50).apply(batch)
    ref = np.stack([ao.vectorize(w) for _, _, w in ao.windower(img000012, 100, 50)]).astype(np.float32)
    assert wins.rows == 15 and np.array_equal(wins.to_numpy(np.float32), ref)
    cc = ks.CenterCornerPatcher(px, py, True).apply(batch)
    ref = np.stack([ao.vectorize(p) for *_, p in ao.center_corner_patcher(img000012, px, py, True)]).astype(np.float32)
    assert np.array_equal(cc.to_numpy(np.float32), ref)
    rp = ks.RandomPatcher(5, px, py).apply(batch)
    ref = np.stack([ao.vectorize(p) for *_, p in ao.random_patcher([img000012], 5, px, py)]).astype(np.float32)
    assert np.array_equal(rp.to_numpy(np.float32), ref)


def test_composed_views_bit_identical(ctx):
    rng = np.random.default_rng(2)
    imgs = rng.integers(0, 256, (4, 32, 32, 3)).astype(np.float32)
    batch = ks.ImageBatch.from_images(ctx, imgs)
    rp = ks.RandomPatcher(3, 24, 24).apply(batch)
    flipped = ks.RandomImageTransformer(0.5, ks.flip_horizontal).apply(rp)
    patches = ao.random_patcher(list(imgs.astype(np.float64)), 3, 24, 24)
    flags, ref_imgs = ao.random_image_transformer([p for *_, p in patches], 0.5)
    assert np.array_equal(flipped.to_numpy(np.float32), np.stack([ao.vectorize(im) for im in ref_imgs]).astype(np.float32))
    # a crop and windows of flipped views are views of the source
    cropped = ks.Cropper(2, 5, 20, 21).apply(flipped)
    ref = np.stack([ao.vectorize(ao.crop(im, 2, 5, 20, 21)) for im in ref_imgs]).astype(np.float32)
    assert np.array_equal(cropped.to_numpy(np.float32), ref)
    wins = ks.Windower(7, 6).apply(flipped)
    ref = np.stack([ao.vectorize(w) for im in ref_imgs for _, _, w in ao.windower(im, 7, 6)]).astype(np.float32)
    assert np.array_equal(wins.to_numpy(np.float32), ref)
    assert list(flipped.views[:, 3]) == flags


def test_image_view_rejections(ctx):
    batch = ks.ImageBatch.from_images(ctx, np.zeros((2, 10, 12, 3), np.float32))
    h = C.c_int64(0)

    def rc(views, ox=4, oy=4, x_dim=10, y_dim=12, ch=3):
        v = np.ascontiguousarray(views, dtype=np.int32).reshape(-1, 4)
        return lib().ks_image_views(ctx.handle, batch.matrix.handle, x_dim, y_dim, ch, v.ctypes.data_as(C.c_void_p), v.shape[0], ox, oy,
                                    C.byref(h))

    assert rc([(1, 6, 8, 1)]) == 0
    for bad in ([(2, 0, 0, 0)], [(-1, 0, 0, 0)], [(0, 7, 0, 0)], [(0, -1, 0, 0)], [(0, 0, 9, 0)], [(0, 0, -1, 0)], [(0, 0, 0, 2)]):
        assert rc(bad) == KS_ERR_INVALID, bad
    assert rc([(0, 0, 0, 0)], ox=0) == KS_ERR_INVALID
    assert rc([(0, 0, 0, 0)], ox=11) == KS_ERR_INVALID
    assert rc([(0, 0, 0, 0)], x_dim=11) == KS_ERR_INVALID
    with pytest.raises(ks.KeystoneError):
        ks.Cropper(0, 0, 11, 4).apply(batch)


# ------------------------------------------------------------------------------------------------------------ Convolver on views
@pytest.mark.parametrize("precision", [2, 1], ids=["parity", "fast"])
def test_convolver_over_views_matches_materialised(ctx, precision):
    rng = np.random.default_rng(3)
    imgs = rng.integers(0, 256, (40, 32, 32, 3)).astype(np.float32)
    batch = ks.ImageBatch.from_images(ctx, imgs)
    views = ks.RandomImageTransformer(0.5, ks.flip_horizontal).apply(ks.RandomPatcher(5, 24, 24).apply(batch))
    mat = views.matrix
    filters = rng.standard_normal((32, 108))
    means = rng.standard_normal(108) * 0.1
    conv = ks.Convolver(ctx, filters, 24, 24, 3, whitener_means=means)
    ctx.set_option("precision", precision)
    try:
        a = conv.apply(views).to_numpy(np.float32)        # unpooled: rows of 19 x 19 x 32 values
        b = conv.apply(mat).to_numpy(np.float32)
        assert np.array_equal(a, b)
        chain = lambda x: ks.ImageVectorizer().apply(ks.Pooler(9, 10).apply(ks.SymmetricRectifier(alpha=0.25).apply(conv.apply(x))))
        pa, pb, pb2 = chain(views).to_numpy(np.float32), chain(mat).to_numpy(np.float32), chain(mat).to_numpy(np.float32)
    finally:
        ctx.set_option("precision", 2)
    # the pooled sums are fp32 atomics in both paths: the two agree as two runs of the materialised path agree
    scale = np.abs(pb).max()
    assert np.abs(pa - pb).max() <= max(4 * np.abs(pb2 - pb).max(), 1e-6 * scale), (np.abs(pa - pb).max(), np.abs(pb2 - pb).max())
    if precision != 2:
        return
    # and in the parity mode the chain over views is the featurizer of the oracle
    ref = ao.features([ao.view_image(imgs[i].astype(np.float64), sx, sy, 24, 24, f) for i, sx, sy, f in views.views], filters, means,
                      0.25, 9, 10)
    assert np.abs(pa - ref).max() <= 1e-4 * np.abs(ref).max()


def test_convolver_views_rejections(ctx):
    batch = ks.ImageBatch.from_images(ctx, np.zeros((2, 32, 32, 3), np.float32))
    conv = ks.Convolver(ctx, np.ones((32, 108)), 24, 24, 3)
    h = C.c_int64(0)
    for views, sx in (([(0, 9, 0, 0)], 32), ([(2, 0, 0, 0)], 32), ([(0, 0, 0, 3)], 32), ([(0, 0, 0, 0)], 31)):
        v = np.ascontiguousarray(views, dtype=np.int32)
        assert lib().ks_convolver_apply_views(ctx.handle, conv._h.handle, batch.matrix.handle, sx, 32, v.ctypes.data_as(C.c_void_p), 1,
                                              9, 10, 0.0, 0.25, C.byref(h)) == KS_ERR_INVALID
    with pytest.raises(ks.KeystoneError):
        conv.apply(ks.Windower(1, 20).apply(batch))


# ------------------------------------------------------------------------------------------------------------- normalizeRows
def test_stats_normalize_rows_within_one_ulp(ctx):
    rng = np.random.default_rng(4)
    X = rng.integers(0, 256, (3000, 108)).astype(np.float32)
    X[5] = 17.0                                              # zero variance
    Y = (rng.standard_normal((500, 333)) * 100 + 5).astype(np.float32)
    for M, alpha in ((X, 10.0), (Y, 1.0), (Y, 0.0)):
        got = ks.stats_normalize_rows(ctx.matrix(M), alpha).to_numpy(np.float32)
        assert _ulps(got, ko.normalize_rows(M.astype(np.float64), alpha).astype(np.float32)).max() <= 1
    one = rng.standard_normal((7, 1)).astype(np.float32)     # one column: the variance is NaN, sd -> sqrt(alpha)
    got = ks.stats_normalize_rows(ctx.matrix(one), 4.0).to_numpy(np.float32)
    assert _ulps(got, ko.normalize_rows(one.astype(np.float64), 4.0).astype(np.float32)).max() <= 1
    h = C.c_int64(0)
    m = ctx.matrix(X[:4])
    assert lib().ks_matrix_stats_normalize_rows(ctx.handle, m.handle, float("nan"), C.byref(h)) == KS_ERR_INVALID


# ------------------------------------------------------------------------------------------------------------- StandardScaler
def test_standard_scaler(ctx):
    rng = np.random.default_rng(5)
    X = (rng.standard_normal((5000, 300)) * rng.uniform(0.1, 50, 300) + rng.uniform(-100, 100, 300)).astype(np.float32)
    X[:, 7] = 3.0                                            # zero std -> 1.0
    x = ctx.matrix(X)
    model = ks.StandardScaler().fit(x)
    mean, std = ko.standard_scaler_fit(X.astype(np.float64))
    assert np.abs(model.mean - mean).max() <= 1e-12 * np.abs(mean).max()
    assert (np.abs(model.std - std) <= 1e-12 * std).all() and model.std[7] == 1.0
    out = model.apply(x).to_numpy(np.float32)
    assert _ulps(out, ko.standard_scaler_apply(X.astype(np.float64), model.mean, model.std).astype(np.float32)).max() <= 1
    again = ks.StandardScaler().fit(x)
    assert np.array_equal(again.mean, model.mean) and np.array_equal(again.std, model.std)
    centred = ks.StandardScaler(normalizeStdDev=False).fit(x)
    assert centred.std is None and np.array_equal(centred.mean, model.mean)
    assert _ulps(centred.apply(x).to_numpy(np.float32), (X.astype(np.float64) - model.mean).astype(np.float32)).max() <= 1
    one = ks.StandardScaler().fit(ctx.matrix(X[:1]))         # one row: variance 0 -> std 1.0
    assert (one.std == 1.0).all()
    # the existing constructor keeps working, with a context given for apply
    assert np.array_equal(ks.StandardScalerModel(model.mean, model.std, ctx).apply(X).to_numpy(np.float32), out)


def test_standard_scaler_rejections(ctx):
    x = ctx.matrix(np.ones((4, 3), np.float32))
    mean, std = np.zeros(3), np.ones(3)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib().ks_standard_scaler_fit(ctx.handle, x.handle, 1, -1.0, p(mean), p(std)) == KS_ERR_INVALID
    assert lib().ks_standard_scaler_fit(ctx.handle, x.handle, 1, float("inf"), p(mean), p(std)) == KS_ERR_INVALID
    assert lib().ks_standard_scaler_fit(ctx.handle, x.handle, 2, 1e-12, p(mean), p(std)) == KS_ERR_INVALID
    h = C.c_int64(0)
    for m, s in ((mean, np.array([1.0, 0.0, 1.0])), (mean, np.array([1.0, np.inf, 1.0])), (np.array([0.0, np.nan, 0.0]), std)):
        assert lib().ks_standard_scaler_apply(ctx.handle, x.handle, p(m), p(s), C.byref(h)) == KS_ERR_INVALID


def _scaler_worker(rank, world, id_holder, ret):
    sys.path.insert(0, ROOT)
    import keystone_b200 as ks
    X = np.random.default_rng(6).standard_normal((3001, 130)).astype(np.float32) * 7 + 2
    lo, hi = ks.shard_range(X.shape[0], rank, world)
    c = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    m = ks.StandardScaler().fit(c.matrix(X[lo:hi]))
    ret[f"mean{rank}"], ret[f"std{rank}"] = m.mean, m.std
    c.close()


def test_two_rank_scaler_equals_one_rank(ctx):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    id_holder, ret = mgr.dict(), mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_scaler_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    X = np.random.default_rng(6).standard_normal((3001, 130)).astype(np.float32) * 7 + 2
    one = ks.StandardScaler().fit(ctx.matrix(X))
    for r in range(2):
        assert np.allclose(ret[f"mean{r}"], one.mean, rtol=1e-12, atol=1e-13)
        assert np.allclose(ret[f"std{r}"], one.std, rtol=1e-12, atol=0)
    assert np.array_equal(ret["mean0"], ret["mean1"]) and np.array_equal(ret["std0"], ret["std1"])


# ---------------------------------------------------------------------------------------------------- AugmentedExamplesEvaluator
@pytest.mark.parametrize("policy", ["average", "borda"])
def test_evaluator_counts_equal_oracle(ctx, policy):
    rng = np.random.default_rng(7)
    n_img, k = 700, 10
    per = rng.integers(1, 12, n_img)
    names = rng.permutation(np.repeat(np.arange(n_img) * 3 + 1, per))   # views of an image are scattered over the rows
    labels_img = rng.integers(0, k, n_img * 3 + 2)
    labels = labels_img[names]
    S = rng.integers(-3, 4, (names.size, k)).astype(np.float32) * 0.5     # many ties within a view and between classes
    S[::7] = 1.0
    got = ks.AugmentedExamplesEvaluator(names, k, policy).evaluate(ctx.matrix(S), labels)
    assert np.array_equal(got.confusionMatrix, ao.augmented_confusion(S, names, labels, k, policy))


def test_evaluator_rejections(ctx):
    S = ctx.matrix(np.zeros((4, 3), np.float32))
    with pytest.raises(ks.KeystoneError):
        ks.AugmentedExamplesEvaluator(["a", "a", "b", "b"], 3).evaluate(S, [0, 1, 2, 2])   # one name, two labels
    with pytest.raises(ks.KeystoneError):
        ks.AugmentedExamplesEvaluator(["a", "a", "b", "b"], 3).evaluate(S, [0, 0, 3, 3])   # label outside [0, k)
    with pytest.raises(ks.KeystoneError):
        ks.AugmentedExamplesEvaluator(["a", "a", "b", "b"], 4).evaluate(S, [0, 0, 1, 1])   # k != score columns
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    out = np.zeros(9)
    lab = np.zeros(4, np.int32)
    for rows, offs, pol in (([0, 1, 1, 3], [0, 2, 4], 0), ([0, 1, 2, 3], [0, 2, 2, 4], 0), ([0, 1, 2, 3], [0, 2, 3], 0),
                            ([0, 1, 2, 3], [0, 2, 4], 2)):
        r, o = np.array(rows, np.int64), np.array(offs, np.int64)
        assert lib().ks_grouped_confusion_matrix(ctx.handle, S.handle, p(r), p(o), o.size - 1, p(lab), 3, pol, p(out)) == KS_ERR_INVALID


# ----------------------------------------------------------------------------------------------------- pipelines in miniature
def _cifar_like(rng, n):
    labels = rng.integers(0, 10, n).astype(np.int32)
    data = rng.integers(0, 200, (n, 3, 32, 32))
    data[:, 0] += labels[:, None, None] * 5                       # a class-dependent colour, so that the classes can be learnt
    return ks.LabeledData(labels=labels, data=data.astype(np.uint8))


def _margin_ok(dev_cm, ref_scores, group_labels, tol):
    """The device confusion matrix equals the oracle's up to the groups whose oracle top-two margin is below tol."""
    pred = ref_scores.argmax(1)
    top2 = np.sort(ref_scores, 1)[:, -2:]
    low = (top2[:, 1] - top2[:, 0]) < tol
    ref_cm = np.zeros_like(dev_cm)
    np.add.at(ref_cm, (group_labels, pred), 1)
    assert np.abs(dev_cm - ref_cm).sum() <= 2 * low.sum(), (np.abs(dev_cm - ref_cm).sum(), low.sum())


@pytest.mark.parametrize("augmented", [False, True], ids=["random_patch_cifar", "random_patch_cifar_augmented"])
def test_pipeline_end_to_end(ctx, augmented):
    rng = np.random.default_rng(8)
    train, test = _cifar_like(rng, 256), _cifar_like(rng, 64)
    conf = pipelines.RandomCifarFeaturizerConfig(numFilters=32, whitenerSize=4096, lam=100.0)
    run = pipelines.random_patch_cifar_augmented if augmented else pipelines.random_patch_cifar
    fitted, train_eval, test_eval = run(ctx, train, test, conf)
    tr_imgs, te_imgs = ao.cifar_images(train.data), ao.cifar_images(test.data)

    # same samples as the oracle; whitener and filters
    n_win = 256 * 27 * 27
    sample_idx = np.random.default_rng(42).choice(n_win, 4096, replace=False)
    filter_idx = np.sort(np.random.default_rng(42).choice(4096, 32, replace=False))
    filters, W, means, _ = ao.learn_filters(tr_imgs, 6, 1, sample_idx, filter_idx, 0.1)
    rel = lambda a, b: np.linalg.norm(a - b) / np.linalg.norm(b)
    assert rel(fitted.whitener, W) <= 1e-6 and rel(fitted.whitener_means, means) <= 1e-6
    assert rel(fitted.filters, filters) <= 1e-6, rel(fitted.filters, filters)

    # the training views and their features
    if augmented:
        patches = ao.random_patcher(tr_imgs, 10, 24, 24)
        flags, views = ao.random_image_transformer([p for *_, p in patches], 0.5)
        dev_views = ks.RandomImageTransformer(0.5, ks.flip_horizontal).apply(
            ks.RandomPatcher(10, 24, 24).apply(ks.ImageBatch.from_images(ctx, np.stack(tr_imgs).astype(np.float32))))
        assert [tuple(v) for v in dev_views.views] == [(i, sx, sy, f) for (i, sx, sy, _), f in zip(patches, flags)]
        train_in, classes = dev_views, np.repeat(train.labels, 10)
        tr_oracle_imgs = views
    else:
        train_in, classes = ks.ImageBatch.from_images(ctx, np.stack(tr_imgs).astype(np.float32)), train.labels
        tr_oracle_imgs = tr_imgs
    stride, size = conf.poolStride, conf.poolSize
    raw_dev = ks.ImageVectorizer().apply(fitted.pooler.apply(fitted.rectifier.apply(fitted.convolver.apply(train_in)))).to_numpy()
    raw_ref = ao.features(tr_oracle_imgs, filters, means, conf.alpha, stride, size)
    assert np.abs(raw_dev - raw_ref).max() <= 1e-4 * np.abs(raw_ref).max()

    # scaler and solver on the device's own features (the pooled sums are fp32 atomics, so a second featurisation differs from the
    # one the pipeline fitted on in the last bits: refit the scaler on the features at hand)
    mean, std = ko.standard_scaler_fit(raw_dev)
    scaler = ks.StandardScaler().fit(ctx.matrix(raw_dev.astype(np.float32)))
    assert np.abs(scaler.mean - mean).max() <= 1e-12 * np.abs(mean).max()
    assert np.abs(scaler.std - std).max() <= 1e-12 * std.max()
    assert rel(fitted.scaler.mean, mean) <= 1e-6 and rel(fitted.scaler.std, std) <= 1e-6
    F_dev = fitted.features(train_in).to_numpy()
    xs, b0, mus = ko.block_ls_fit(F_dev, ko.class_label_indicators(classes, 10), 4096, 1, conf.lam)
    W_dev, W_ref = np.concatenate(fitted.model.xs, 0), np.concatenate(xs, 0)
    assert rel(W_dev, W_ref) <= 1e-4, rel(W_dev, W_ref)
    assert train_eval.confusionMatrix.sum() == classes.size

    # test metrics against the all-oracle pipeline, up to low-margin examples
    xs_o, b_o, mus_o, mean_o, std_o = ao.fit_predict(raw_ref, classes, conf.lam)
    if augmented:
        te_views = [ao.view_image(im, sx, sy, 24, 24, f) for im in te_imgs for sx, sy, f, _ in ao.center_corner_patcher(im, 24, 24, True)]
        s_ref = ko.block_linear_apply(ko.standard_scaler_apply(ao.features(te_views, filters, means, conf.alpha, stride, size), mean_o, std_o),
                                      xs_o, 4096, b_o, mus_o)
        dev_views = ks.CenterCornerPatcher(24, 24, True).apply(ks.ImageBatch.from_images(ctx, np.stack(te_imgs).astype(np.float32)))
        s_dev = fitted.apply(dev_views).to_numpy()
        names = np.repeat(np.arange(64), 10)
        assert np.array_equal(test_eval.confusionMatrix, ao.augmented_confusion(s_dev, names, np.repeat(test.labels, 10), 10))
        g_ref = s_ref.reshape(64, 10, 10).mean(1)
        tol = 2 * np.abs(s_dev - s_ref).max()
    else:
        s_ref = ko.block_linear_apply(ko.standard_scaler_apply(ao.features(te_imgs, filters, means, conf.alpha, stride, size), mean_o, std_o),
                                      xs_o, 4096, b_o, mus_o)
        s_dev = fitted.apply(ks.ImageBatch.from_images(ctx, np.stack(te_imgs).astype(np.float32))).to_numpy()
        g_ref = s_ref
        tol = 2 * np.abs(s_dev - s_ref).max()
    assert tol <= 1e-2 * np.abs(s_ref).max()
    _margin_ok(test_eval.confusionMatrix, g_ref, test.labels, tol)
