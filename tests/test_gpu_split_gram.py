"""One-pass split-operand Gram (parity mode, fp16 pairs): ks_debug_gram with context precision KS_PRECISION_F16X2 splits the fp32
operands into fp16 pairs hi + lo and runs the split kernel, which must return G = A^T A (upper tiles, symmetrised) and C = A^T B as
hi^T hi + lo^T hi + hi^T lo.

The operands are built so that every partial sum is exact in fp32: hi holds small nonzero integers and lo = j * 2^-14 with a small
integer j.  The only rounding left is the fp32 sum of the two accumulators and the fp32 reduce-add of the row chunks, so the bound sits at
the fp32 level of the combined sum; a wrong descriptor, swizzle, plane or tile mask moves entries by O(1) (hi) or by the size of
the cross terms (lo), both far above it."""
import ctypes as C

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import check, lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    c.set_option("precision", 2)  # KS_PRECISION_F16X2: the debug entry runs the split kernel
    yield c
    c.close()


def _pair_operand(rng, n, m):
    # nonzero integers and |lo| < 2^-12 (half an fp16 step just below 1): fp16(hi + lo) is hi itself, so the device's split
    # recovers exactly these planes and hi^T hi is an exact integer sum
    hi = rng.integers(1, 4, (n, m)).astype(np.float64) * rng.choice([-1.0, 1.0], (n, m))
    lo = rng.integers(-3, 4, (n, m)).astype(np.float64) * 2.0 ** -14
    return hi + lo


def _split(v):
    """What the device does: hi = fp16(v), lo = fp16(v - hi)."""
    hi = v.astype(np.float32).astype(np.float16).astype(np.float64)
    lo = (v.astype(np.float32) - hi.astype(np.float32)).astype(np.float16).astype(np.float64)
    return hi, lo


def _debug_gram(ctx, A, B):
    a, b = ctx.matrix(A.astype(np.float32)), ctx.matrix(B.astype(np.float32))
    m, kc = A.shape[1], B.shape[1]
    G = np.zeros((m, m))
    Cm = np.zeros((m, kc))
    check(ctx.handle, lib().ks_debug_gram(ctx.handle, a.handle, b.handle, G.ctypes.data_as(C.c_void_p), m,
                                          Cm.ctypes.data_as(C.c_void_p), kc))
    return G, Cm


def _check(G, ref, hi_a, hi_b, lo_a, lo_b, n_chunks):
    # every partial sum is exact; each fp32 addition of a chunk's (hh + cross) and of the chunks into the output rounds once
    mag = np.abs(hi_a).T @ np.abs(hi_b) + np.abs(hi_a).T @ np.abs(lo_b) + np.abs(lo_a).T @ np.abs(hi_b)
    tol = (2 * n_chunks + 1) * 2.0 ** -24 * mag + 1e-12
    err = np.abs(G - ref)
    assert (err <= tol).all(), (err.max(), np.unravel_index(np.argmax(err - tol), err.shape))


# columns not a multiple of 128, rows not a multiple of the chunk or of the 32-row stage, a single output column
@pytest.mark.parametrize("n,m,kc,chunk", [(777, 200, 70, 0), (5000, 130, 1, 0), (1000, 300, 37, 96), (333, 64, 129, 32),
                                          (4173, 257, 1000, 0)])
def test_split_gram_matches_fp64_pair_products(ctx, n, m, kc, chunk):
    rng = np.random.default_rng(n + m + kc)
    A = _pair_operand(rng, n, m)
    B = _pair_operand(rng, n, kc)
    ah, al = _split(A)
    bh, bl = _split(B)
    assert np.array_equal(ah, np.round(A)) and np.array_equal(bh, np.round(B))
    ctx.set_option("gram_chunk_rows", chunk)
    try:
        G, Cm = _debug_gram(ctx, A, B)
    finally:
        ctx.set_option("gram_chunk_rows", 0)
    n_chunks = -(-n // (chunk or 4096))
    g_ref = ah.T @ ah + al.T @ ah + ah.T @ al
    c_ref = ah.T @ bh + al.T @ bh + ah.T @ bl
    # the test only means something if the cross terms are far above the bound
    assert np.abs(g_ref - ah.T @ ah).max() > 1e-3 and np.abs(c_ref - ah.T @ bh).max() > 1e-3
    _check(G, g_ref, ah, ah, al, al, n_chunks)
    _check(Cm, c_ref, ah, bh, al, bl, n_chunks)
