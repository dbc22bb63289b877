"""The CIFAR random-patch pipelines of the reference on the device (K/pipelines/images/cifar/RandomPatchCifar.scala,
RandomPatchCifarAugmented.scala), DESIGN.md section 21, and the text pipelines (K/pipelines/text/AmazonReviewsPipeline.scala,
NewsgroupsPipeline.scala), DESIGN.md section 23.

Filter learning: ``Windower -> ImageVectorizer -> Sampler(whitenerSize) -> Stats.normalizeRows(., 10) -> ZCAWhitenerEstimator ->
sampleRows(numFilters) -> whiten -> unit norm -> . whitener^T``.  Everything with a row per window, view or image runs on the device;
only the numFilters x patch arithmetic of the last three steps runs in fp64 NumPy, as it does on the reference's driver.  Single
rank: the augmented evaluation groups views by image, and a group must not span ranks.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

from .context import Context, DeviceMatrix
from .evaluation import AugmentedExamplesEvaluator, BinaryClassifierEvaluator, MulticlassClassifierEvaluator
from .nodes import (CommonSparseFeatures, LogisticRegressionEstimator, LowerCase, MaxClassifier, NaiveBayesEstimator, NGramsFeaturizer,
                    TermFrequency, Tokenizer, Trim)
from .nodes import (BlockLeastSquaresEstimator, BlockLinearMapper, CenterCornerPatcher, Convolver, ImageBatch, ImageVectorizer, Pooler,
                    RandomImageTransformer, RandomPatcher, Sampler, StandardScaler, StandardScalerModel, SymmetricRectifier, Windower,
                    ZCAWhitenerEstimator, cifar_bytes_to_matrix, flip_horizontal, sample_rows, stats_normalize_rows)

NUM_CLASSES = 10
NUM_CHANNELS = 3
IMAGE_SIZE = 32
AUGMENT_IMAGE_SIZE = 24
FLIP_CHANCE = 0.5
NUM_TEST_AUGMENT = 10   # the four corners and the centre, each with its flip


@dataclass
class RandomCifarFeaturizerConfig:
    """``RandomCifarFeaturizerConfig``'s defaults (RandomPatchCifarAugmented.scala:108-120) without the file locations and
    ``sampleFrac``.  ``whitenerSize`` is the reference's constant 100000 (the patches the whitener is fitted on)."""
    numFilters: int = 100
    whiteningEpsilon: float = 0.1
    patchSize: int = 6
    patchSteps: int = 1
    poolSize: int = 10
    poolStride: int = 9
    alpha: float = 0.25
    lam: Optional[float] = None
    numRandomImagesAugment: int = 10
    whitenerSize: int = 100000


@dataclass
class RandomPatchCifarModel:
    """The fitted ``Convolver -> SymmetricRectifier -> Pooler -> ImageVectorizer -> StandardScalerModel -> BlockLinearMapper``."""
    convolver: Convolver
    rectifier: SymmetricRectifier
    pooler: Pooler
    scaler: StandardScalerModel
    model: BlockLinearMapper
    filters: np.ndarray      # numFilters x patch, packFilters order, whitened
    whitener: np.ndarray     # patch x patch
    whitener_means: np.ndarray

    def features(self, images) -> DeviceMatrix:
        """Scaled features of an ImageBatch or of ImageViews."""
        raw = ImageVectorizer().apply(self.pooler.apply(self.rectifier.apply(self.convolver.apply(images))))
        return self.scaler.apply(raw)

    def apply(self, images) -> DeviceMatrix:
        """Class scores (BlockLinearMapper.apply) of every image or view."""
        return self.model.apply(self.features(images))


def _train_images(ctx: Context, data) -> ImageBatch:
    """CifarLoader's records (n, 3, 32, 32) as an ImageBatch."""
    return ImageBatch(ctx.matrix(cifar_bytes_to_matrix(np.asarray(data))), IMAGE_SIZE, IMAGE_SIZE, NUM_CHANNELS)


def learn_filters(ctx: Context, images: ImageBatch, conf: RandomCifarFeaturizerConfig):
    """(filters, whitener, whitener means) as RandomPatchCifar.scala:41-58 computes them."""
    patches = Sampler(conf.whitenerSize).apply(Windower(conf.patchSteps, conf.patchSize).apply(images))
    base = stats_normalize_rows(patches.matrix, 10.0)
    zca = ZCAWhitenerEstimator(eps=conf.whiteningEpsilon).fit_single(base)
    W, means = zca.whitener, zca.means
    sample = sample_rows(base, conf.numFilters).to_numpy(np.float64)
    unnorm = (sample - means) @ W
    norms = np.sqrt((unnorm ** 2).sum(axis=1))
    return (unnorm / (norms + 1e-10)[:, None]) @ W.T, W, means


def _fit(ctx: Context, train_images, train_classes: np.ndarray, filters, W, means, size: int, conf: RandomCifarFeaturizerConfig):
    conv = Convolver(ctx, filters, size, size, NUM_CHANNELS, whitener_means=means, normalize_patches=True)
    rect, pool = SymmetricRectifier(alpha=conf.alpha), Pooler(conf.poolStride, conf.poolSize)
    raw = ImageVectorizer().apply(pool.apply(rect.apply(conv.apply(train_images))))
    scaler = StandardScaler().fit(raw)
    feats = scaler.apply(raw)
    labels = ctx.labels_from_classes(train_classes, NUM_CLASSES)
    model = BlockLeastSquaresEstimator(4096, 1, conf.lam or 0.0).fit(feats, labels)
    train_eval = MulticlassClassifierEvaluator(NUM_CLASSES).evaluate_model(model, feats, labels)
    return RandomPatchCifarModel(conv, rect, pool, scaler, model, filters, W, means), train_eval


def _single_rank(ctx: Context) -> None:
    if ctx.world_size > 1:
        raise NotImplementedError("the CIFAR and text pipelines run on one rank")


def random_patch_cifar(ctx: Context, train, test, conf: Optional[RandomCifarFeaturizerConfig] = None):
    """``RandomPatchCifar.run``: train and test are ``LabeledData`` as ``CifarLoader`` returns them.  Returns (fitted model, train
    metrics, test metrics)."""
    _single_rank(ctx)
    conf = conf or RandomCifarFeaturizerConfig()
    images = _train_images(ctx, train.data)
    filters, W, means = learn_filters(ctx, images, conf)
    fitted, train_eval = _fit(ctx, images, np.asarray(train.labels), filters, W, means, IMAGE_SIZE, conf)
    feats = fitted.features(_train_images(ctx, test.data))
    test_eval = MulticlassClassifierEvaluator(NUM_CLASSES).evaluate_model(fitted.model, feats,
                                                                          ctx.labels_from_classes(np.asarray(test.labels), NUM_CLASSES))
    return fitted, train_eval, test_eval


def random_patch_cifar_augmented(ctx: Context, train, test, conf: Optional[RandomCifarFeaturizerConfig] = None):
    """``RandomPatchCifarAugmented.run``: the model is fitted on ``numRandomImagesAugment`` random 24 x 24 crops per training image,
    each flipped with chance 0.5, and tested on the ten ``CenterCornerPatcher(24, 24, true)`` views per test image, scored by
    ``AugmentedExamplesEvaluator`` (average policy).  Returns (fitted model, train metrics over the training views, test
    metrics)."""
    _single_rank(ctx)
    conf = conf or RandomCifarFeaturizerConfig()
    images = _train_images(ctx, train.data)
    filters, W, means = learn_filters(ctx, images, conf)
    n_aug = conf.numRandomImagesAugment
    train_views = RandomImageTransformer(FLIP_CHANCE, flip_horizontal).apply(
        RandomPatcher(n_aug, AUGMENT_IMAGE_SIZE, AUGMENT_IMAGE_SIZE).apply(images))
    train_classes = np.repeat(np.asarray(train.labels), n_aug)          # LabelAugmenter
    fitted, train_eval = _fit(ctx, train_views, train_classes, filters, W, means, AUGMENT_IMAGE_SIZE, conf)
    test_images = _train_images(ctx, test.data)
    test_views = CenterCornerPatcher(AUGMENT_IMAGE_SIZE, AUGMENT_IMAGE_SIZE, True).apply(test_images)
    names = np.repeat(np.arange(test_images.rows), NUM_TEST_AUGMENT)
    scores = fitted.apply(test_views)
    test_eval = AugmentedExamplesEvaluator(names, NUM_CLASSES).evaluate(scores, np.repeat(np.asarray(test.labels), NUM_TEST_AUGMENT))
    return fitted, train_eval, test_eval


# ------------------------------------------------------------------------------------------ text pipelines (DESIGN.md section 23)
@dataclass
class AmazonReviewsConfig:
    """``AmazonReviewsConfig``'s defaults without the file locations and ``numParts``."""
    threshold: float = 3.5
    nGrams: int = 2
    commonFeatures: int = 100000
    numIters: int = 20


@dataclass
class NewsgroupsConfig:
    nGrams: int = 2
    commonFeatures: int = 100000


def _one(x):
    return 1.0


def _text_featurizer(ctx: Context, train_docs, n_grams: int, common_features: int):
    """``Trim andThen LowerCase() andThen Tokenizer() andThen NGramsFeaturizer(1 to n) andThen TermFrequency(x => 1) andThen
    (CommonSparseFeatures(k), train)``"""
    return (Trim(ctx=ctx).andThen(LowerCase()).andThen(Tokenizer()).andThen(NGramsFeaturizer(range(1, n_grams + 1)))
            .andThen(TermFrequency(_one)).andThen(CommonSparseFeatures(common_features), train_docs))


def amazon_reviews_pipeline(ctx: Context, train, test, conf: Optional[AmazonReviewsConfig] = None):
    """``AmazonReviewsPipeline.run``: train and test are ``LabeledData`` as ``AmazonReviewsDataLoader`` returns them.  Logistic
    regression (2 classes, ``numIters``) on the common n-gram features; returns (fitted predictor, test
    ``BinaryClassificationMetrics`` of prediction > 0 against label > 0)."""
    _single_rank(ctx)
    conf = conf or AmazonReviewsConfig()
    train_docs = ctx.text(list(train.data))
    labels = np.asarray(train.labels)
    predictor = _text_featurizer(ctx, train_docs, conf.nGrams, conf.commonFeatures).andThen(
        LogisticRegressionEstimator(num_classes=2, num_iters=conf.numIters), train_docs, labels).fit()
    results = predictor(ctx.text(list(test.data)))
    return predictor, BinaryClassifierEvaluator.evaluate(np.asarray(results) > 0, np.asarray(test.labels) > 0)


def newsgroups_pipeline(ctx: Context, train, test, conf: Optional[NewsgroupsConfig] = None):
    """``NewsgroupsPipeline.run``: train and test are ``LabeledData`` as ``NewsgroupsDataLoader`` returns them.  Naive Bayes over the
    20 classes, then ``MaxClassifier``; returns (fitted predictor, test ``MulticlassMetrics``)."""
    from .loaders import NewsgroupsDataLoader
    _single_rank(ctx)
    conf = conf or NewsgroupsConfig()
    k = len(NewsgroupsDataLoader.classes)
    train_docs = ctx.text(list(train.data))
    predictor = _text_featurizer(ctx, train_docs, conf.nGrams, conf.commonFeatures).andThen(
        NaiveBayesEstimator(k), train_docs, np.asarray(train.labels)).andThen(MaxClassifier()).fit()
    pred = np.asarray(predictor(ctx.text(list(test.data))))
    cm = np.zeros((k, k), dtype=np.float64)
    np.add.at(cm, (np.asarray(test.labels, dtype=np.int64), pred.astype(np.int64)), 1.0)
    return predictor, MulticlassClassifierEvaluator.from_confusion_matrix(cm)
