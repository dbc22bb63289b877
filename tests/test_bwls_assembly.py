"""The algebra of the device's BlockWeightedLeastSquares, without a GPU: bwls_oracle.device_assembly_fit rebuilds H, rhs and
finalB from the statistics of the SHIFTED blocks, as bwls.cu does, and must equal the reference restatement
(keystone_oracle.bwls_fit) to fp64 rounding for any shift.  When a device test of the weighted solver fails, this test tells a
wrong formula (fails here too) apart from device arithmetic (passes here)."""
import os
import sys

import numpy as np
import pytest

from oracle import keystone_oracle as ko

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bwls_oracle as bo  # noqa: E402

TOL = 1e-10


def _shifts(rng):
    return {
        "zero": lambda blk: np.zeros(blk.shape[1]),
        "population_mean": lambda blk: blk.mean(axis=0),
        # a crude estimate, as the sampled mean of generated features is: a few rows, plus an offset
        "crude": lambda blk: blk[::7].mean(axis=0) + 0.3 * rng.standard_normal(blk.shape[1]),
    }


def _check(F, Y, bs, iters, lam, w, shift, nf=None):
    xs_d, fb_d, _ = bo.device_assembly_fit(F, Y, bs, iters, lam, w, shift, nf)
    xs_r, fb_r = ko.bwls_fit(F, Y, bs, iters, lam, w, num_features=nf)
    assert [x.shape for x in xs_d] == [x.shape for x in xs_r]
    Wd, Wr = np.concatenate(xs_d, 0), np.concatenate(xs_r, 0)
    assert np.linalg.norm(Wd - Wr) <= TOL * max(np.linalg.norm(Wr), 1.0), np.linalg.norm(Wd - Wr)
    assert np.abs(fb_d - fb_r).max() <= TOL * max(np.abs(fb_r).max(), 1.0)


@pytest.mark.parametrize("shift", ["zero", "population_mean", "crude"])
@pytest.mark.parametrize("bs,iters", [(4, 10), (5, 3), (12, 1)])
def test_assembly_matches_oracle_on_reference_fixture(golden_dir, shift, bs, iters):
    A = np.loadtxt(os.path.join(golden_dir, "aMat.csv"), delimiter=",")
    B = np.loadtxt(os.path.join(golden_dir, "bMat.csv"), delimiter=",")
    _check(A, B, bs, iters, 0.1, 0.3, _shifts(np.random.default_rng(bs))[shift])


@pytest.mark.parametrize("shift", ["zero", "population_mean", "crude"])
@pytest.mark.parametrize("seed,n,d,k,bs,iters,w,nf", [
    (1, 400, 37, 6, 16, 3, 0.25, None),     # ragged last block, interleaved classes
    (2, 300, 40, 9, 40, 2, 0.75, 33),       # num_features < D, one block
    (3, 500, 24, 12, 7, 2, 0.5, None),      # empty classes (k > classes drawn)
])
def test_assembly_matches_oracle_on_random_problems(shift, seed, n, d, k, bs, iters, w, nf):
    rng = np.random.default_rng(seed)
    # class centroids apart and a common offset: the shift matters to the arithmetic, never to the algebra
    cls = rng.integers(0, k - 2 if seed == 3 else k, n)
    cent = 3.0 * rng.standard_normal((k, d))
    F = cent[cls] + rng.standard_normal((n, d)) + 5.0
    Y = ko.class_label_indicators(cls, k)
    _check(F, Y, bs, iters, 0.5, w, _shifts(rng)[shift], nf)


def test_assembled_systems_equal_reference_systems(golden_dir):
    """The first-sweep (H, rhs) of every class rebuilt from shifted statistics equal jointXTX + lambda I and jointXTR built
    from raw features (rhs: block 0 only, where the residual does not depend on earlier solves)."""
    rng = np.random.default_rng(4)
    n, d, k = 600, 50, 5
    cls = rng.integers(0, k, n)
    F = 2.0 * rng.standard_normal((k, d))[cls] + rng.standard_normal((n, d)) + 50.0
    Y = ko.class_label_indicators(cls, k)
    _, _, systems = bo.device_assembly_fit(F, Y, 20, 1, 0.2, 0.25, lambda blk: blk[:50].mean(axis=0))
    for j in range(3):
        ref = bo.reference_systems(F, Y, 20, 0.2, 0.25, j)
        for c, (H, rhs) in ref.items():
            Hd, rd = systems[(j, c)]
            assert np.abs(Hd - H).max() <= 1e-9 * np.abs(H).max()
            if j == 0:
                assert np.abs(rd - rhs).max() <= 1e-9 * np.abs(rhs).max()


def test_class_ranges_follow_a_stable_class_sort():
    Y = ko.class_label_indicators(np.array([2, 0, 2, 3, 0, 0]), 5)
    perm, ranges = bo.class_ranges(Y)
    assert list(perm) == [1, 4, 5, 0, 2, 3]
    assert ranges == [(0, 0, 3), (2, 3, 2), (3, 5, 1)]
