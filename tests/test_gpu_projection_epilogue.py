"""The slab producers' asynchronous epilogue (gemm_kmajor_kernel with a separate epilogue warpgroup) and the exact Gram diagonal
it accumulates for the parity mode's fp16 pairs.

ks_debug_time_slab launches produce_slab as a block fit's first sweep does (on the look-ahead stream, column sums on, for the fp16
pair also the fp64 diagonal) and returns the slab and diagonal of its last launch; the option reserve_sms sets how many SMs that
launch leaves free.
"""
import ctypes as C

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import KS_PRECISION_F16, KS_PRECISION_F16X2, KS_PRECISION_TF32, check, lib

pytestmark = pytest.mark.gpu

TILE = 128


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def n_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _timed_slab(ctx, x, rfs, prec, round_out, rows, cols, reserve=None):
    arr = (C.c_int64 * len(rfs))(*[r.handle for r in rfs])
    pair = prec == KS_PRECISION_F16X2
    out = np.zeros((rows, cols))
    lo = np.zeros((rows, cols)) if pair else None
    diag = np.zeros(cols) if pair else None
    ms = C.c_double()
    if reserve is not None:
        ctx.set_option("reserve_sms", reserve)
    try:
        check(ctx.handle, lib().ks_debug_time_slab(ctx.handle, x.handle, arr, len(rfs), prec, round_out, cols, 1, C.byref(ms),
                                                   _ptr(diag), _ptr(out), _ptr(lo)))
    finally:
        ctx.set_option("reserve_sms", 8)
    return out, lo, diag


def _maps(ctx, rng, n, d_in, widths):
    X = rng.standard_normal((n, d_in)).astype(np.float32)
    rfs = [ks.CosineRandomFeatures(ctx, rng.standard_normal((m, d_in)) * 0.3, rng.random(m) * 2 * np.pi) for m in widths]
    return ctx.matrix(X), rfs


@pytest.mark.parametrize("rows,widths,cols", [(1000, (100, 60, 90), 250), (333, (97,), 97), (4133, (300, 200), 500)])
def test_diagonal_matches_the_stored_pair(ctx, rows, widths, cols):
    """The epilogue's diagonal is the fp64 sum of (hi + lo)^2 over exactly the stored rows: row counts with rows % 32 != 0 and a
    column tail, so padding rows (where the cosine of the bias alone is far from zero) would show in it."""
    rng = np.random.default_rng(rows)
    x, rfs = _maps(ctx, rng, rows, 40, widths)
    assert rows % 32 != 0 and cols % 32 != 0
    hi, lo, diag = _timed_slab(ctx, x, rfs, KS_PRECISION_F16X2, 0, rows, cols)
    ref = ((hi + lo) ** 2).sum(0)
    assert np.all(ref > 0)
    np.testing.assert_allclose(diag, ref, rtol=1e-12, atol=0)
    # one leaked padding row would add about 0.5 per column on average, far above the tolerance
    assert 0.1 > 1e-12 * ref.max()


@pytest.mark.parametrize("kind", ["tf32", "f16", "f16x2_pair"])
def test_slab_independent_of_the_schedule(ctx, n_sms, kind):
    """At least 9 tiles per CTA on 1, 2 and all SMs, with K = 40 (one stage per tile) and with the split operands' 3 d_in = 120:
    the slab is bitwise the same whichever CTA took which tile and however far the epilogue warpgroup trailed the MMA."""
    prec, round_out = {"tf32": (KS_PRECISION_TF32, 1), "f16": (KS_PRECISION_F16, 1), "f16x2_pair": (KS_PRECISION_F16X2, 0)}[kind]
    rng = np.random.default_rng(7)
    rows, cols = 3 * 128 - 50, 3 * 128 - 20     # 9 tiles, both edges partial
    x, rfs = _maps(ctx, rng, rows, 40, (cols,))
    results = {}
    for ctas in (1, 2, n_sms):
        results[ctas] = _timed_slab(ctx, x, rfs, prec, round_out, rows, cols, reserve=n_sms - ctas)
    base = results[1]
    assert np.abs(base[0]).max() > 0
    for ctas, res in results.items():
        for a, b in zip(base[:2], res[:2]):   # the planes; the diagonal's fp64 atomics follow the tile order
            if a is not None:
                assert np.array_equal(a, b), (kind, ctas)
        if base[2] is not None:
            np.testing.assert_allclose(res[2], base[2], rtol=1e-12, atol=0)


def test_many_tiles_per_cta(ctx, n_sms):
    """All SMs with more than 8 tiles each (the tile-id ring's depth): pair, column tail and a partial last row tile."""
    rng = np.random.default_rng(9)
    rows, cols = (9 * n_sms + 1) * TILE - 50, 200
    x, rfs = _maps(ctx, rng, rows, 40, (cols,))
    hi, lo, diag = _timed_slab(ctx, x, rfs, KS_PRECISION_F16X2, 0, rows, cols, reserve=0)
    hi1, lo1, diag1 = _timed_slab(ctx, x, rfs, KS_PRECISION_F16X2, 0, rows, cols, reserve=n_sms - 1)
    assert np.array_equal(hi, hi1) and np.array_equal(lo, lo1)
    np.testing.assert_allclose(diag, ((hi + lo) ** 2).sum(0), rtol=1e-12, atol=0)
    np.testing.assert_allclose(diag1, diag, rtol=1e-12, atol=0)


def test_diagonal_only_for_the_pair(ctx):
    rng = np.random.default_rng(3)
    x, rfs = _maps(ctx, rng, 256, 40, (64,))
    arr = (C.c_int64 * 1)(rfs[0].handle)
    ms = C.c_double()
    diag = np.zeros(64)
    rc = lib().ks_debug_time_slab(ctx.handle, x.handle, arr, 1, KS_PRECISION_F16, 1, 64, 1, C.byref(ms), _ptr(diag), None, None)
    assert rc != 0
