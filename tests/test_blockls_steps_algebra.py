"""CPU companion of tests/test_gpu_blockls_steps.py: the step algebra of the block least-squares fit (shift, delta, the rank-1
correction, rhs with -delta rsum^T - lambda W_old, the update with cbias) restated in numpy reproduces the fp64 oracle for any
shift, and the reference and bound functions the GPU test applies to captured states accept a correctly computed step and
reject one that misses a term."""
import os
import sys

import numpy as np
import pytest

from oracle import keystone_oracle as ko

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blockls_steps_ref as st  # noqa: E402


@pytest.mark.parametrize("iters", [1, 2, 3])
def test_restated_fit_reproduces_the_oracle(iters):
    """Shift from the first rows of class-sorted data (far from the mean: a large delta), ragged last block."""
    rng = np.random.default_rng(iters)
    n, d, k, bs, lam = 700, 90, 4, 32, 3.0
    cls = np.sort(rng.integers(0, k, n))
    F = rng.standard_normal((n, d)) + 2.0 * rng.standard_normal((k, d))[cls]
    Y = ko.class_label_indicators(cls, k)
    bounds = ko.block_bounds(d, bs)
    assert bounds[-1][1] - bounds[-1][0] == 26
    shifts = [st.shift_estimate(F[:, s:e], 37) for s, e in bounds]
    assert max(np.abs(F[:, s:e].mean(0) - m).max() for (s, e), m in zip(bounds, shifts)) > 0.5
    xs, ybar, means = st.restated_fit(F, Y, bs, iters, lam, shifts)
    rxs, rybar, rmeans = ko.block_ls_fit(F, Y, bs, iters, lam)
    W, R = np.concatenate(xs, 0), np.concatenate(rxs, 0)
    assert np.abs(W - R).max() <= 1e-10 * np.abs(R).max()
    assert np.abs(ybar - rybar).max() <= 1e-12
    assert np.abs(np.concatenate(means) - np.concatenate(rmeans)).max() <= 1e-12


def test_split_formats():
    rng = np.random.default_rng(1)
    v = (rng.standard_normal((300, 20)) * 10.0 ** rng.integers(-6, 4, (300, 20))).astype(np.float32)
    hi, lo = st.center_round(v, np.zeros(20), pair=True)
    assert (np.abs(hi + lo - v) <= 2.0 ** -22 * np.abs(v)).all()
    assert np.array_equal(hi, st.round_tf32(hi)) and np.array_equal(lo, st.round_tf32(lo))
    hi1, lo1 = st.center_round(v, np.zeros(20), pair=False)
    assert (np.abs(hi1 - v) <= 2.0 ** -11 * np.abs(v)).all() and not lo1.any()
    s = 2.0 ** np.floor(np.log2(4096.0 / np.abs(v).max()))   # the device's choice: largest magnitude into [2048, 4096]
    h, l = st.fp16_pair(v, s)
    assert (np.abs(h + l - v) <= st.operand_error(v, "f16x2", s)).all()


def _step_problem(mode, seed=3):
    """A generated-like block (values of order 1, shift from 64 of 3000 rows) in the device's operand format."""
    rng = np.random.default_rng(seed)
    n, b, k, lam = 3000, 40, 6, 50.0
    cls = np.sort(rng.integers(0, k, n))
    F = np.cos(rng.standard_normal((n, b)) + 0.8 * rng.standard_normal((k, b))[cls])
    shift = st.shift_estimate(F, 64)
    pair, f16, _ = st.MODES[mode]
    if f16:
        v = (F - shift).astype(np.float32)
        hi, lo = st.fp16_pair(v, 1.0) if pair else (v.astype(np.float16).astype(np.float64), np.zeros_like(F))
    else:
        hi, lo = st.center_round(F, shift, pair)
    S = hi + lo
    delta = S.mean(0)
    R = (ko.class_label_indicators(cls, k) - 1.0 / k).astype(np.float32).astype(np.float64)
    W_old = 0.05 * rng.standard_normal((b, k))
    return hi, lo, delta, R, lam, W_old


def _f32(x):
    return np.asarray(x).astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("mode", list(st.MODES))
def test_bounds_accept_a_correct_step_and_reject_missing_terms(mode):
    hi, lo, delta, R, lam, W_old = _step_problem(mode)
    n = hi.shape[0]
    chain = 4096
    S = hi + lo
    H = st.system(hi, lo, delta, lam)
    bH = st.system_bound(hi, lo, delta, lam, mode, chain)
    # a device-like H: the Gram rounded to fp32 (off the diagonal unless the diagonal is exact), assembled in fp64
    G = S.T @ S
    Gd = _f32(G)
    if st.MODES[mode][2]:
        np.fill_diagonal(Gd, np.diag(G))
    Hd = Gd - n * np.outer(delta, delta) + lam * np.eye(len(delta))
    assert st.ratio(np.abs(Hd - H), bH) <= 1
    assert st.ratio(np.abs(Hd + n * np.outer(delta, delta) - H), bH) > 1          # N delta delta^T dropped
    assert st.ratio(np.abs(Hd - lam * np.eye(len(delta)) - H), bH) > 1          # lambda dropped
    if st.MODES[mode][2]:   # the tensor core's diagonal: its truncating chain sits low by ~chain / 16 ulps
        biased = Hd - np.diag((chain / 16) * 2.0 ** -24 * np.diag(G))
        assert st.ratio(np.abs(biased - H), bH) > 1
    rhs = st.rhs_of(hi, lo, delta, R, lam, W_old)
    bR = st.rhs_bound(hi, lo, delta, R, lam, W_old, mode, chain, 1.0)
    assert st.ratio(np.abs(_f32(S.T @ R) - np.outer(delta, R.sum(0)) - lam * W_old - rhs), bR) <= 1
    assert st.ratio(np.abs(rhs + lam * W_old - rhs), bR) > 1                     # lambda W_old dropped
    Rs = R + 0.25   # a residual that is not centred: the -delta rsum^T term is then far above the bound
    assert st.ratio(np.abs(st.rhs_of(hi, lo, delta, Rs, lam, None) + np.outer(delta, Rs.sum(0)) - st.rhs_of(hi, lo, delta, Rs, lam, None)),
                    st.rhs_bound(hi, lo, delta, Rs, lam, None, mode, chain, 1.0)) > 1
    dW = np.linalg.solve(H, rhs)
    assert st.ratio(np.abs(H @ dW - rhs), st.solve_bound(H, dW)) <= 1
    assert st.ratio(np.abs(H @ _f32(dW) - rhs), st.solve_bound(H, dW)) > 1           # an fp32 solve is far outside
    Ra = st.update_of(hi, lo, delta, R, dW)
    bU = st.update_bound(hi, lo, delta, R, dW, mode, 1.0)
    assert st.ratio(np.abs(_f32(Ra) - Ra), bU) <= 1
    assert st.ratio(np.abs(Ra - delta @ dW - Ra), bU) > 1                          # cbias dropped
    m = S.mean(0)
    assert (np.abs(_f32(S.sum(0)) / n - m) <= st.delta_bound(hi, lo)).all()
    assert (np.abs(delta) > 100 * st.delta_bound(hi, lo)).any()
