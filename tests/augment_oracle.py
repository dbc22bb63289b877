"""fp64 NumPy restatement of the CIFAR random-patch front end and of test-time augmentation, written from the reference's Scala and
independently of keystone_b200/nodes.py:
  java.util.Random                  the JDK's 48-bit LCG, nextInt(), nextInt(bound), nextDouble()
  Windower / crop / flipHorizontal  K/nodes/images/Windower.scala, K/utils/images/ImageUtils.scala (crop, flipHorizontal)
  RandomPatcher, CenterCornerPatcher, RandomImageTransformer   K/nodes/images/*.scala
  AugmentedExamplesEvaluator        K/evaluation/AugmentedExamplesEvaluator.scala
  the two CIFAR pipelines           K/pipelines/images/cifar/RandomPatchCifar{,Augmented}.scala, composed from the existing oracles
Images are (x, y, c) arrays; ImageVectorizer order is value (x, y, c) at c + x C + y C xDim.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import keystone_oracle as ko  # noqa: E402
import pca_oracle as po  # noqa: E402


def _int32(v: int) -> int:
    v &= 0xFFFFFFFF
    return v - 0x100000000 if v & 0x80000000 else v


class JdkRandom:
    """java.util.Random as the JDK documents it (setSeed scrambles with 0x5DEECE66D; next(bits) = (int)(seed >>> (48 - bits)))."""

    def __init__(self, seed: int):
        self.state = (seed ^ 0x5DEECE66D) % (1 << 48)

    def next_bits(self, bits: int) -> int:
        self.state = (self.state * 0x5DEECE66D + 11) % (1 << 48)
        return _int32(self.state >> (48 - bits))

    def next_int(self, bound=None) -> int:
        if bound is None:
            return self.next_bits(32)
        r = self.next_bits(31)
        m = bound - 1
        if (bound & m) == 0:
            return _int32((bound * r) >> 31)
        u = r
        while True:
            r = u % bound
            if _int32(u - r + m) >= 0:      # Java's int arithmetic: the sum overflows to a negative value for the rejected draws
                return r
            u = self.next_bits(31)

    def next_double(self) -> float:
        hi = self.next_bits(26)
        lo = self.next_bits(27)
        return float(hi * (1 << 27) + lo) / float(1 << 53)


def vectorize(img: np.ndarray) -> np.ndarray:
    return ko.image_vectorizer(img)


def crop(img: np.ndarray, sx: int, sy: int, ex: int, ey: int) -> np.ndarray:
    xd, yd = img.shape[0], img.shape[1]
    if sx < 0 or sx > xd or ex < 0 or ex > xd or sy < 0 or sy > yd or ey < 0 or ey > yd or sx > ex or sy > ey:
        raise ValueError("invalid crop")
    out = np.zeros((ex - sx, ey - sy, img.shape[2]))
    for x in range(sx, ex):
        for y in range(sy, ey):
            out[x - sx, y - sy, :] = img[x, y, :]
    return out


def flip_horizontal(img: np.ndarray) -> np.ndarray:
    """ImageUtils.flipHorizontal: res(x, yDim - 1 - y, c) = im(x, y, c)."""
    yd = img.shape[1]
    out = np.zeros_like(img, dtype=np.float64)
    for y in range(yd):
        out[:, yd - 1 - y, :] = img[:, y, :]
    return out


def windower(img: np.ndarray, stride: int, w: int):
    """[(x, y, window)] for x outer, y inner."""
    xd, yd = img.shape[0], img.shape[1]
    return [(x, y, crop(img, x, y, x + w, y + w)) for x in range(0, xd - w + 1, stride) for y in range(0, yd - w + 1, stride)]


def random_patcher(images, n: int, px: int, py: int, seed: int = 12334):
    """[(image index, startX, startY, patch)] over all images in order, one generator for the call."""
    rnd = JdkRandom(seed)
    out = []
    for i, img in enumerate(images):
        for _ in range(n):
            sx = rnd.next_int(img.shape[0] - px + 1)
            sy = rnd.next_int(img.shape[1] - py + 1)
            out.append((i, sx, sy, crop(img, sx, sy, sx + px, sy + py)))
    return out


def center_corner_patcher(img: np.ndarray, px: int, py: int, flips: bool):
    """[(startX, startY, flipped, patch)] in the reference's order."""
    xd, yd = img.shape[0], img.shape[1]
    sxs = [0, xd - px, 0, xd - px, (xd - px) // 2]
    sys_ = [0, 0, yd - py, yd - py, (yd - py) // 2]
    out = []
    for sx, sy in zip(sxs, sys_):
        im = crop(img, sx, sy, sx + px, sy + py)
        out.append((sx, sy, 0, im))
        if flips:
            out.append((sx, sy, 1, flip_horizontal(im)))
    return out


def random_image_transformer(images, chance: float, seed: int = 12334):
    """(flags, images): flags[i] = 1 where the flip applied."""
    rnd = JdkRandom(seed)
    flags, out = [], []
    for im in images:
        f = rnd.next_double() < chance
        flags.append(int(f))
        out.append(flip_horizontal(im) if f else im)
    return flags, out


def borda(vec: np.ndarray) -> np.ndarray:
    order = sorted(range(len(vec)), key=lambda i: vec[i])          # Python's sort is stable, as Scala's sortBy
    rank = np.zeros(len(vec))
    for pos, cls in enumerate(order):
        rank[cls] = pos
    return rank


def augmented_confusion(scores: np.ndarray, names, labels, k: int, policy: str = "average") -> np.ndarray:
    groups = {}
    for v, name in enumerate(names):
        groups.setdefault(name, []).append(v)
    cm = np.zeros((k, k))
    for views in groups.values():
        lab = {int(labels[v]) for v in views}
        assert len(lab) == 1
        if policy == "average":
            agg = np.zeros(k)
            for v in views:
                agg = agg + scores[v].astype(np.float64)
            agg = agg / len(views)
        else:
            agg = np.zeros(k)
            for v in views:
                agg = agg + borda(scores[v])
        cm[lab.pop(), int(np.argmax(agg))] += 1
    return cm


# ------------------------------------------------------------------------------------------------------------- the pipelines
def cifar_images(records: np.ndarray):
    """CifarLoader records (n, 3, 32, 32) as (x, y, c) images."""
    return [np.transpose(r, (1, 2, 0)).astype(np.float64) for r in np.asarray(records)]


def window_rows(images, stride: int, w: int) -> np.ndarray:
    """Windower andThen ImageVectorizer over a list of images, by slicing (the loops of crop are too slow for many windows)."""
    return np.stack([vectorize(img[x:x + w, y:y + w, :]) for img in images for x in range(0, img.shape[0] - w + 1, stride)
                     for y in range(0, img.shape[1] - w + 1, stride)])


def view_image(img: np.ndarray, sx: int, sy: int, px: int, py: int, flip: int) -> np.ndarray:
    v = img[sx:sx + px, sy:sy + py, :]
    return v[:, ::-1, :] if flip else v


def learn_filters(images, patch_size: int, patch_steps: int, sample_idx, filter_idx, eps: float):
    """RandomPatchCifar.scala:41-58 with the Sampler's and sampleRows' row choices given."""
    wins = window_rows(images, patch_steps, patch_size)
    base = ko.normalize_rows(wins[np.asarray(sample_idx)], 10.0)
    W, means = po.zca_fit(base, eps)
    unnorm = (base[np.asarray(filter_idx)] - means) @ W
    norms = np.sqrt((unnorm ** 2).sum(axis=1))
    return (unnorm / (norms + 1e-10)[:, None]) @ W.T, W, means, base


def features(images, filters, means, alpha: float, pool_stride: int, pool_size: int) -> np.ndarray:
    return np.stack([ko.random_patch_cifar_features(im, filters, means, 6, alpha, pool_stride, pool_size) for im in images])


def fit_predict(train_feats: np.ndarray, train_classes, lam: float, k: int = 10):
    """StandardScaler -> BlockLeastSquaresEstimator(4096, 1, lam): (xs, label mean, feature means, scaler mean, scaler std)."""
    mean, std = ko.standard_scaler_fit(train_feats)
    F = ko.standard_scaler_apply(train_feats, mean, std)
    xs, b, mus = ko.block_ls_fit(F, ko.class_label_indicators(np.asarray(train_classes), k), 4096, 1, lam)
    return xs, b, mus, mean, std
