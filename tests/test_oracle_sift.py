"""The NumPy SIFT oracle (tests/sift_oracle.py) against the reference's own output on images/000012.jpg (feats128.csv, the
descriptors of SIFTExtractor(scaleStep = 0) after PixelScaler and GrayScaler), the SIFTExtractorSuite property, and the host-only
keypoint geometry of the C ABI.  The fixture keeps the zero / nonzero status of all 64 990 keypoints and the full descriptors of
every 32nd (tests/golden/make_sift_golden.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import sift_oracle as so  # noqa: E402


@pytest.fixture(scope="module")
def fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "sift_000012.npz"))
    return z["rgb"], z["zero"], z["cols"], z["feats"]


@pytest.fixture(scope="module")
def oracle_000012(fixture):
    rgb = fixture[0]
    return so.sift_extract(so.gray_f32(rgb), 3, 4, 4, 0, with_mass=True)


def test_fixture_counts_and_order(fixture, oracle_000012):
    """vlfeat's per-scale counts for the 333 x 500 image add up to the fixture's 64 990 columns, and scale 0's zero mask agrees
    position by position with frames in the order vlfeat-y (160) outer, x (104) inner."""
    rgb, zero, cols, feats = fixture
    assert rgb.shape == (333, 500, 3) and zero.shape == (64990,) and feats.shape == (128, cols.size)
    assert np.array_equal(zero[cols], (feats == 0).all(0))
    assert so.keypoint_counts(333, 500, 3, 4, 4, 0) == [16640, 16377, 16116, 15857]
    D, _ = oracle_000012
    assert D.shape == (64990, 128)
    assert (zero[:16640] == (D[:16640] == 0).all(1)).mean() > 0.999


def test_oracle_matches_feats128(fixture, oracle_000012):
    """The restatement against the reference's numbers: >= 99.5 % of keypoints with the same zero / nonzero status, and among
    keypoints nonzero in both >= 99 % of entries within 1 and >= 95 % exact (measured on all 64 990 keypoints: 99.99 %, 100 %,
    99.99 %).  The status is compared on every keypoint, the entries on the sampled ones."""
    _, zero, cols, feats = fixture
    D, _ = oracle_000012
    zd = (D == 0).all(1)
    assert (zero == zd).mean() >= 0.995
    ref, Ds = feats.T.astype(np.float32), D[cols]
    both = ~zero[cols] & ~zd[cols]
    assert both.sum() > 500
    diff = np.abs(Ds[both] - ref[both])
    assert (diff <= 1).mean() >= 0.99
    assert (diff == 0).mean() >= 0.95
    assert D.min() >= 0 and D.max() <= 255 and np.array_equal(D, np.floor(D))


def test_nonzero_descriptors_are_512_unit_vectors(oracle_000012):
    D, _ = oracle_000012
    nz = D[(D != 0).any(1)]
    norms = np.linalg.norm(nz, axis=1)
    assert 480 < norms.min() and norms.max() <= 512.5


def test_scale_step_one_gives_fewer_descriptors():
    """SIFTExtractorSuite: scaleStep = 1 gives fewer descriptors than scaleStep = 0 on 000012.jpg's shape."""
    assert sum(so.keypoint_counts(333, 500, 3, 4, 4, 1)) < sum(so.keypoint_counts(333, 500, 3, 4, 4, 0))


def test_transpose_is_a_permutation():
    p = so.transpose_perm()
    assert sorted(p.tolist()) == list(range(128))
    # output j = 8 (y + 4 x) + tT takes raw 8 (x + 4 y) + (10 - tT) % 8 (the closed form the device kernel uses)
    j = np.arange(128)
    closed = 8 * ((j >> 5) + 4 * ((j >> 3) & 3)) + ((10 - (j & 7)) & 7)
    assert np.array_equal(p, closed)


def test_negative_offset_is_clamped_to_zero():
    """scales = 5: off = 11 - 3 s is -1 at s = 4; vl_dsift_set_bounds clamps the minimum to 0."""
    geo = so.scale_geometry(100, 90, 3, 4, 5, 1)
    assert [g[2] for g in geo] == [11, 8, 5, 2, 0]
    b, st = 4 + 8, 3 + 4
    assert geo[4][3] == ((100 - 1) - 0 - 3 * b) // st + 1 and geo[4][4] == ((90 - 1) - 0 - 3 * b) // st + 1


def test_scales_without_frames():
    """30 x 30 at the defaults: 3 x 3 frames, 2 x 2, exactly 1, and none at the last scale."""
    counts = so.keypoint_counts(30, 30, 3, 4, 4, 1)
    assert counts == [9, 4, 1, 0]
    D = so.sift_extract(np.random.default_rng(0).random((30, 30)).astype(np.float32), 3, 4, 4, 1)
    assert D.shape == (sum(counts), 128)


def test_triangle_filter_matches_direct_convolution():
    """The running-sum triangle equals the direct convolution with max(F - |t|, 0) / F^2 and continuity padding."""
    rng = np.random.default_rng(1)
    a = rng.random((23, 3)).astype(np.float32)
    for F in (1, 4, 9, 30):
        got = so.conv_col_tri(a, F).astype(np.float64)
        idx = np.arange(23)
        want = np.zeros((23, 3))
        for t in range(-F + 1, F):
            want += (F - abs(t)) / F ** 2 * a[np.clip(idx + t, 0, 22)].astype(np.float64)
        assert np.allclose(got, want, rtol=1e-5, atol=1e-6)


def test_gray_conversion_is_rounded_once():
    rgb = np.random.default_rng(2).integers(0, 256, size=(7, 5, 3), dtype=np.uint8)
    g = so.gray_f32(rgb)
    r, gg, b = (rgb[:, :, k].astype(np.float64) / 255.0 for k in range(3))
    assert np.array_equal(g, (0.2989 * r + 0.5870 * gg + 0.1140 * b).astype(np.float32))


# ------------------------------------------------------------------------------------------------------ host-only C ABI
@pytest.fixture(scope="module")
def lib():
    from keystone_b200 import _capi
    if not os.path.exists(_capi.LIB_PATH):
        from keystone_b200 import build
        build.build(verbose=False)
    return _capi.lib()


@pytest.mark.parametrize("args", [(333, 500, 3, 4, 4, 0), (333, 500, 3, 4, 4, 1), (500, 375, 3, 4, 4, 0), (40, 40, 3, 4, 4, 1),
                                  (100, 90, 3, 4, 5, 1), (13, 13, 1, 4, 1, 0), (12, 13, 1, 4, 1, 0), (61, 47, 2, 3, 3, 2)])
def test_sift_keypoints_matches_oracle(lib, args):
    counts = np.full(args[4], -1, dtype=np.int64)
    assert lib.ks_sift_keypoints(*args, counts.ctypes.data_as(C.POINTER(C.c_int64))) == 0
    assert counts.tolist() == so.keypoint_counts(*args)


@pytest.mark.parametrize("args", [(0, 10, 3, 4, 4, 1), (10, -1, 3, 4, 4, 1), (10, 10, 0, 4, 4, 1), (10, 10, 3, 0, 4, 1),
                                  (10, 10, 3, 4, 0, 1), (10, 10, 3, 4, 4, -1)])
def test_sift_keypoints_rejects(lib, args):
    counts = np.zeros(8, dtype=np.int64)
    assert lib.ks_sift_keypoints(*args, counts.ctypes.data_as(C.POINTER(C.c_int64))) == -1


def test_sift_nodes_are_exported_and_shaped():
    import keystone_b200 as ks
    from keystone_b200 import _capi
    for name in ("ks_image_pixel_scale", "ks_image_grayscale", "ks_sift_extract", "ks_sift_keypoints"):
        assert name in _capi.declared_symbols()
    se = ks.SIFTExtractor()
    assert (se.step, se.bin, se.scales, se.scale_step) == (3, 4, 4, 1) and se.descriptorSize == 128
    assert se.keypoints(333, 500) == sum(so.keypoint_counts(333, 500, 3, 4, 4, 1))
    with pytest.raises(ks.KeystoneError):
        ks.SIFTExtractor(stepSize=0).keypoints(50, 50)
