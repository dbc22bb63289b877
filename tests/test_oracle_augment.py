"""CPU checks of tests/augment_oracle.py against the reference suites (WindowingSuite, CenterCornerPatcherSuite, RandomPatcherSuite),
the JDK's java.util.Random values, hand cases of AugmentedExamplesEvaluator, and the product's host-side view tables and generator
against the oracle's."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import augment_oracle as ao  # noqa: E402

import keystone_b200 as ks  # noqa: E402
from keystone_b200 import nodes  # noqa: E402


def _scala_image(arr, x_dim, y_dim, ch):
    """ChannelMajorArrayVectorizedImage(arr, ImageMetadata(x_dim, y_dim, ch)) as an (x, y, c) array."""
    arr = np.asarray(arr, dtype=np.float64)
    return arr.reshape(y_dim, x_dim, ch).transpose(1, 0, 2)


def _suite_array(dim_x, dim_y, fn):
    """The suites' (0 until X).flatMap(x => (0 until Y).flatMap(y => (0 until 1).map(c => fn(x, y, c)))) array."""
    return [fn(x, y, 0) for x in range(dim_x) for y in range(dim_y)]


@pytest.fixture(scope="module")
def img000012(golden_dir):
    """images/000012.jpg as (x, y, c) values (the shape is what these suites check)."""
    return np.load(os.path.join(golden_dir, "sift_000012.npz"))["rgb"].astype(np.float64)


# ------------------------------------------------------------------------------------------------------------ WindowingSuite
def test_windowing_1x1():
    img = _scala_image(_suite_array(4, 4, lambda x, y, c: c + x + y * 4), 4, 4, 1)
    wins = ao.windower(img, 1, 1)
    assert len(wins) == 16
    assert [w[2][0, 0, 0] for w in wins[:4]] == [0.0, 1.0, 2.0, 3.0]


def test_windowing_2x2():
    img = _scala_image(_suite_array(4, 4, lambda x, y, c: c + x + y * 4), 4, 4, 1)
    wins = ao.windower(img, 2, 2)
    assert [w[2][0, 0, 0] for w in wins] == [0.0, 2.0, 8.0, 10.0]


def test_windowing_real_image(img000012):
    wins = ao.windower(img000012, 100, 50)
    assert all(w[2].shape[:2] == (50, 50) for w in wins)
    assert len(wins) == (img000012.shape[0] // 100) * (img000012.shape[1] // 100) == 15


@pytest.mark.parametrize("w", [1, 2, 3, 4, 6, 8])
def test_windowing_nxn(w):
    dim = 30
    img = _scala_image(_suite_array(dim, dim, lambda x, y, c: c + x + y * 4 + 10), dim, dim, 1)
    wins = ao.windower(img, 1, w)
    assert len(wins) == (dim - w + 1) ** 2
    assert all((win != 0).all() for _, _, win in wins)


# ---------------------------------------------------------------------------------------------------- CenterCornerPatcherSuite
def test_center_corner_1x1():
    img = _scala_image(_suite_array(5, 5, lambda x, y, c: c + x + y * 5), 5, 5, 1)
    got = [p[3][0, 0, 0] for p in ao.center_corner_patcher(img, 1, 1, False)]
    assert got == [0.0, 20.0, 4.0, 24.0, 12.0]


def test_center_corner_real_image(img000012):
    px, py = img000012.shape[0] // 2, img000012.shape[1] // 2
    for flips, count in ((True, 10), (False, 5)):
        ps = ao.center_corner_patcher(img000012, px, py, flips)
        assert len(ps) == count
        assert all(p[3].shape == (px, py, 3) for p in ps)
    ps = ao.center_corner_patcher(img000012, px, py, True)
    assert np.array_equal(ps[1][3], ps[0][3][:, ::-1, :])           # the flip reverses y


# --------------------------------------------------------------------------------------------------------- RandomPatcherSuite
def test_random_patcher_real_image(img000012):
    px, py = img000012.shape[0] // 2, img000012.shape[1] // 2
    ps = ao.random_patcher([img000012], 5, px, py)
    assert len(ps) == 5
    assert all(p[3].shape == (px, py, 3) for p in ps)


# ------------------------------------------------------------------------------------------------------------ java.util.Random
def test_jdk_random_known_values():
    assert ao.JdkRandom(42).next_int() == -1170105035
    assert ao.JdkRandom(42).next_double() == 0.7275636800328681


@pytest.mark.parametrize("bound", [9, 1, 2, 8, 27, 1 << 30, (1 << 30) + 1, 2147483647])
def test_product_java_random_matches_oracle(bound):
    a, b = ks.JavaRandom(12334), ao.JdkRandom(12334)
    assert [a.nextInt(bound) for _ in range(200)] == [b.next_int(bound) for _ in range(200)]
    assert [a.nextDouble() for _ in range(50)] == [b.next_double() for _ in range(50)]
    assert [a.nextInt() for _ in range(50)] == [b.next_int() for _ in range(50)]


def test_product_java_random_seed_12334():
    r = ks.JavaRandom(12334)
    assert [r.nextInt(9) for _ in range(10)] == [4, 7, 4, 7, 2, 6, 7, 5, 5, 6]


# ---------------------------------------------------------------------------------------------- product view tables on the host
def test_product_view_tables_match_oracle():
    x_dim, y_dim = 32, 30
    imgs = [np.zeros((x_dim, y_dim, 3)) for _ in range(3)]
    rp = nodes.RandomPatcher(4, 24, 20).views(3, x_dim, y_dim)
    assert [tuple(v[:3]) for v in rp] == [(i, sx, sy) for i, sx, sy, _ in ao.random_patcher(imgs, 4, 24, 20)]
    cc = nodes.CenterCornerPatcher(24, 20, True).views(1, x_dim, y_dim)
    assert [tuple(v[1:]) for v in cc] == [(sx, sy, f) for sx, sy, f, _ in ao.center_corner_patcher(imgs[0], 24, 20, True)]
    wv = nodes.Windower(3, 6).views(1, x_dim, y_dim)
    assert [tuple(v[1:3]) for v in wv] == [(x, y) for x, y, _ in ao.windower(imgs[0], 3, 6)]
    flags, _ = ao.random_image_transformer(imgs * 4, 0.5)
    assert list(nodes.RandomImageTransformer(0.5, ks.flip_horizontal).flips(12)) == flags


def test_random_image_transformer_rejects_other_transforms():
    with pytest.raises(ks.KeystoneError):
        nodes.RandomImageTransformer(0.5, lambda im: im)


# ------------------------------------------------------------------------------------------------- AugmentedExamplesEvaluator
def test_borda_ties_go_by_class_index():
    assert list(ao.borda(np.array([1.0, 1.0, 0.0]))) == [1.0, 2.0, 0.0]
    assert list(ao.borda(np.array([2.0, 2.0, 2.0]))) == [0.0, 1.0, 2.0]


def test_evaluator_hand_cases():
    scores = np.array([[0.0, 1.0, 0.5],     # image a: ranks [0, 2, 1]
                       [3.0, 0.0, 0.0],     # image a: ranks [2, 0, 1]
                       [0.2, 0.2, 0.1],     # image b: ranks [1, 2, 0]
                       [0.0, 0.0, 0.0]])    # image b: ranks [0, 1, 2]
    names, labels = ["a", "a", "b", "b"], [1, 1, 2, 2]
    # average: a -> [1.5, 0.5, 0.25] -> 0; b -> [0.1, 0.1, 0.05] -> 0 (first maximum)
    assert np.array_equal(ao.augmented_confusion(scores, names, labels, 3, "average"), [[0, 0, 0], [1, 0, 0], [1, 0, 0]])
    # borda: a -> [2, 2, 2] -> 0; b -> [1, 3, 2] -> 1
    assert np.array_equal(ao.augmented_confusion(scores, names, labels, 3, "borda"), [[0, 0, 0], [1, 0, 0], [0, 1, 0]])


def test_evaluator_groups_by_first_appearance():
    ev = ks.AugmentedExamplesEvaluator(np.array([7, 3, 7, 5, 3]), 2)
    rows, offsets = ev.groups()
    assert list(rows) == [0, 2, 1, 4, 3] and list(offsets) == [0, 2, 4, 5]
