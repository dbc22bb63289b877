"""The K-major tensor-core GEMM (gemm_kmajor_kernel) and its epilogues, each instantiation against an fp64 reference.

ks_debug_update runs launch_update (EPI_UPDATE / EPI_APPLY) and ks_debug_slab runs produce_slab (EPI_COS) exactly as the fits
call them; the pooled Convolver (EPI_POOL) is reached through the public API.  As in test_gpu_split_gram.py the operands are
chosen so that every partial sum is exact in fp32 (small integers, power-of-two scales), and then the results must be bitwise
equal to the reference.  Where a transcendental or a rounded output makes exactness impossible the bound is derived from the
arithmetic of the epilogue, and each such test also asserts that the error it guards against (a row or column off by one, a
missing cross term, a padding row leaked into the column sums) is far above the bound.

Instantiations of gemm_kmajor_kernel<EPI, F16, OUT16, SPLIT> that launch_kmajor selects, and the tests that reach them:
  <UPDATE, tf32, 0>, <APPLY, tf32, 0>, <UPDATE, f16, 0>, <APPLY, f16, 0>, <UPDATE, f16, 0, split>
                                 test_update_and_apply_match_fp64, test_update_wraps_the_tile_ring
  <COS, tf32, 0> (unrounded and tf32-rounded), <COS, tf32, 1> (proj_f16 = 0) and <COS, f16, 1> (each with the __cosf and the
  range-reduced cosine), <COS, f16, 0> (split operands, fp32 slab), <COS, f16, 2> (split operands, fp16 pair)
                                 test_projection_cosine, test_projection_rectified, test_projection_wraps_the_tile_ring
  <POOL, f16, 0>                 test_pooled_convolver_is_exact
  <RBF, f16, 2>                  test_gpu_kernel_ridge.py
"""
import ctypes as C

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import KS_PRECISION_F16, KS_PRECISION_F16X2, KS_PRECISION_TF32, check, lib
from oracle import keystone_oracle as ko

pytestmark = pytest.mark.gpu

W_TOL = 1e-4        # parity mode (tests/test_gpu_parity.py)
W_TOL_FAST = 1.5e-3  # 10-bit operand modes
KS_ERR_INVALID = -1
ACC_SCALE = 2.0 ** -3
EPS32 = 2.0 ** -24   # unit roundoff of fp32
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


def round_tf32(x):
    """fp32 -> tf32 with round-to-nearest (ties away), kept in fp32: what cvt.rna.tf32.f32 does on the device."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def _split16(v):
    """The split-operand copies of an fp32 matrix: scaled by the device's power of two (largest magnitude into [2048, 4096]),
    hi = fp16(v s), lo = fp16(v s - hi), returned unscaled."""
    v32 = np.asarray(v, dtype=np.float32)
    m = float(np.abs(v32).max())
    s = np.float32(2.0 ** np.floor(np.log2(4096.0 / m)))
    if m * s > 4096:
        s /= 2
    hi = (v32 * s).astype(np.float16)
    lo = (v32 * s - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64) / s, lo.astype(np.float64) / s


# ------------------------------------------------------------------------------------------ update and apply (launch_update)
def _update(ctx, A, B, apply, precision, bias, reduce, init):
    a, b = ctx.matrix(A.astype(np.float32)), ctx.matrix(B.astype(np.float32))
    out = ctx.matrix(init.astype(np.float32))
    bp = None if bias is None else np.ascontiguousarray(bias, dtype=np.float64)
    rc = lib().ks_debug_update(ctx.handle, a.handle, b.handle, int(apply), precision, _ptr(bp), int(reduce), ACC_SCALE, out.handle)
    check(ctx.handle, rc)
    return out.to_numpy()


def _pair_operand(rng, n, k):
    """hi: nonzero integers; lo = j 2^-14, |lo| < half an fp16 step of hi: the device's split recovers exactly these planes.
    Row 0 has the largest hi and lo of one sign, so the cross terms of out[0, 0] cannot cancel."""
    hi = rng.integers(1, 4, (n, k)) * rng.choice([-1.0, 1.0], (n, k))
    lo = rng.integers(-3, 4, (n, k)) * 2.0 ** -14
    hi[0], lo[0] = 3.0, 3 * 2.0 ** -14
    return hi, lo


def _check_update(ctx, M, N, K, mode, seed, combos=((0, 0), (0, 1), (1, 0), (1, 1))):
    rng = np.random.default_rng(seed)
    init = rng.integers(-8, 9, (M, N)) * 2.0 ** -3
    bias = rng.integers(-5, 6, N).astype(np.float64)
    if mode != "f16x2":
        prec = KS_PRECISION_TF32 if mode == "tf32" else KS_PRECISION_F16
        A, B = rng.integers(-3, 4, (M, K)).astype(np.float64), rng.integers(-3, 4, (N, K)).astype(np.float64)
        acc = A @ B.T   # integers far below 2^24: every partial sum of the tensor core is exact
        for apply, reduce in combos:
            out = _update(ctx, A, B, apply, prec, bias, reduce, init)
            ref = (init if reduce else 0.0) + bias + (1.0 if apply else -1.0) * ACC_SCALE * acc
            assert np.array_equal(out, ref), (apply, reduce, np.abs(out - ref).max())
        out = _update(ctx, A, B, 0, prec, None, 0, init)   # no bias vector: the epilogue reads zeros
        assert np.array_equal(out, -ACC_SCALE * acc), np.abs(out + ACC_SCALE * acc).max()
        return
    ah, al = _pair_operand(rng, M, K)
    bh, bl = _pair_operand(rng, N, K)
    hh = ah @ bh.T                # exact integers: the hi x hi accumulator
    cross = al @ bh.T + ah @ bl.T  # multiples of 2^-14 below 2^10: the cross accumulator, also exact
    mag = np.abs(ah) @ np.abs(bh).T + np.abs(al) @ np.abs(bh).T + np.abs(ah) @ np.abs(bl).T
    for _, reduce in combos:   # fp16 pairs: residual update only
        out = _update(ctx, ah + al, bh + bl, 0, KS_PRECISION_F16X2, bias, reduce, init)
        ref = (init if reduce else 0.0) + bias - ACC_SCALE * (hh + cross)
        # fp32 roundings left: hh + cross, bias - s acc, the reduce-add; where none of them rounds the result must be exact
        r1 = _f32(hh + cross)
        emul = _f32(bias - ACC_SCALE * r1)
        if reduce:
            emul = _f32(init + emul)
        tol = 3 * EPS32 * ((np.abs(init) if reduce else 0.0) + np.abs(bias) + ACC_SCALE * mag)
        hi_only = (init if reduce else 0.0) + bias - ACC_SCALE * hh
        assert np.abs(ref - hi_only).max() > 10 * tol.max()   # a dropped cross product is far above the bound
        if np.array_equal(emul, ref):
            assert np.array_equal(out, ref), (reduce, np.abs(out - ref).max())
        else:
            err = np.abs(out - ref)
            assert (err <= tol).all(), (reduce, err.max(), np.unravel_index(np.argmax(err - tol), err.shape))
        assert not np.array_equal(out, hi_only)


# M (rows), N (classes), K (block size): tails of the 128 x 128 tile, of the 32-column store chunk and of the K steps of the
# tf32 (32), fp16 (64) and pair (32) stages
UPDATE_SHAPES = [(1, 7, 1), (63, 1, 31), (64, 31, 32), (65, 32, 33), (129, 33, 63), (1000, 129, 64), (4097, 257, 65),
                 (1000, 1000, 200), (63, 257, 200), (4097, 1, 33), (129, 1000, 1), (65, 7, 64), (64, 129, 65), (1, 1000, 63),
                 (4097, 32, 31)]


@pytest.mark.parametrize("mode", ["tf32", "f16", "f16x2"])
@pytest.mark.parametrize("M,N,K", UPDATE_SHAPES)
def test_update_and_apply_match_fp64(ctx, M, N, K, mode):
    combos = ((0, 0), (0, 1), (1, 0), (1, 1)) if mode != "f16x2" else ((0, 0), (0, 1))
    _check_update(ctx, M, N, K, mode, seed=M * 7919 + N * 131 + K, combos=combos)


@pytest.mark.parametrize("mode", ["tf32", "f16", "f16x2"])
def test_update_wraps_the_tile_ring(ctx, n_sms, mode):
    """At least 9 tiles per CTA (static schedule: the update never draws from a counter): the 8-slot tile ring wraps and its
    barrier phase flips."""
    N, K = 129, 32
    n_tiles = 2
    m_tiles = -(-9 * n_sms // n_tiles)
    M = m_tiles * TILE - 5
    total = -(-M // TILE) * n_tiles
    assert -(-total // min(total, n_sms)) >= 9
    _check_update(ctx, M, N, K, mode, seed=17, combos=((0, 1),))


def test_update_rejects_pairs_for_apply(ctx):
    A = np.ones((64, 32))
    a, b, out = ctx.matrix(A), ctx.matrix(A), ctx.matrix(np.zeros((64, 64)))
    rc = lib().ks_debug_update(ctx.handle, a.handle, b.handle, 1, KS_PRECISION_F16X2, None, 0, ACC_SCALE, out.handle)
    assert rc == KS_ERR_INVALID
    rc = lib().ks_debug_update(ctx.handle, a.handle, b.handle, 0, KS_PRECISION_TF32, None, 0, 0.3, out.handle)
    assert rc == KS_ERR_INVALID   # acc_scale must be a power of two


# ------------------------------------------------------------------------------------------ projection (produce_slab, EPI_COS)
# mode -> (precision, round_out, fp16 pair, proj_f16)
SLAB_MODES = {
    "tf32": (KS_PRECISION_TF32, 0, False, 1),             # <COS, tf32, 0>, unrounded (Cody-Waite + __cosf)
    "tf32_rounded": (KS_PRECISION_TF32, 1, False, 1),     # <COS, tf32, 0>, tf32-rounded (__cosf)
    "f16": (KS_PRECISION_F16, 1, False, 1),               # <COS, f16, 1> (__cosf): the fp16-mode blocks
    "f16_tf32_operands": (KS_PRECISION_F16, 1, False, 0),  # <COS, tf32, 1> (__cosf)
    "f16_unrounded": (KS_PRECISION_F16, 0, False, 1),     # <COS, f16, 1>, range-reduced cosine: the fp16-mode mean estimates
    "f16_unrounded_tf32_operands": (KS_PRECISION_F16, 0, False, 0),  # <COS, tf32, 1>, range-reduced cosine
    "f16x2": (KS_PRECISION_F16X2, 0, False, 1),           # <COS, f16, 0>
    "f16x2_pair": (KS_PRECISION_F16X2, 0, True, 1),       # <COS, f16, 2>
}


def _slab(ctx, x, handles, mode, row_begin, rows, c0, cols, shift=None):
    prec, round_out, pair, proj_f16 = SLAB_MODES[mode]
    arr = (C.c_int64 * len(handles))(*handles)
    out = np.zeros((rows, cols))
    lo = np.zeros((rows, cols)) if pair else None
    cs = np.zeros(cols)
    sh = None if shift is None else np.ascontiguousarray(shift, dtype=np.float64)
    ctx.set_option("proj_f16", proj_f16)
    try:
        check(ctx.handle, lib().ks_debug_slab(ctx.handle, x.handle, arr, len(handles), prec, round_out, row_begin, rows, c0, cols,
                                              _ptr(sh), _ptr(out), _ptr(lo), cols, _ptr(cs)))
    finally:
        ctx.set_option("proj_f16", 1)
    return out, lo, cs


def _output_tol(mode, val):
    """Rounding of the stored value: tf32 / fp16 round to 11 significant bits, the pair keeps ~22."""
    prec, round_out, pair, _ = SLAB_MODES[mode]
    if prec == KS_PRECISION_F16 or (prec == KS_PRECISION_TF32 and round_out):
        return 2.0 ** -11 * np.abs(val) + 2.0 ** -25
    if pair:
        return 2.0 ** -22 * np.abs(val) + 2.0 ** -25
    return 0.0


def _check_stored(mode, out, lo):
    if mode == "tf32_rounded":   # the low 13 mantissa bits of every value are zero
        assert not (out.astype(np.float32).view(np.uint32) & np.uint32(0x1FFF)).any()
    if SLAB_MODES[mode][0] == KS_PRECISION_F16:
        assert np.array_equal(out, out.astype(np.float16).astype(np.float64))
    if mode == "f16x2_pair":
        # hi = fp16(hi + lo): lo is the remainder of the split, at most half the gap to hi's neighbour on lo's side.  When the
        # remainder rounds up to exactly that half gap, hi + lo is a tie, which fp16 may resolve away from hi.
        h16 = out.astype(np.float16)
        assert np.array_equal(out, h16.astype(np.float64)) and np.array_equal(lo, lo.astype(np.float16).astype(np.float64))
        gap = np.abs(np.nextafter(h16, np.where(lo >= 0, np.inf, -np.inf).astype(np.float16)).astype(np.float64) - out)
        assert (np.abs(lo) <= gap / 2).all()
        tie = np.abs(lo) == gap / 2
        assert np.array_equal(h16[~tie], (out + lo)[~tie].astype(np.float16))


def _check_colsums(cs, stored, pad_value, rows, leak_measurable=True):
    """Column sums: those of the stored values up to the fp32 order of the chunk sums and atomics; padding rows (past the last
    valid row of the last 128-row tile) evaluate to pad_value and must not be in them."""
    n_chunks = -(-rows // 32)
    tol = (32 + n_chunks) * EPS32 * np.abs(stored).sum(0) + 1e-30
    err = np.abs(cs - stored.sum(0))
    assert (err <= tol).all(), (err.max(), np.argmax(err - tol))
    pad = -(-rows // TILE) * TILE - rows
    assert pad > 0
    if leak_measurable:   # a leaked padding row is far above the bound
        assert np.abs(pad * pad_value).max() > 10 * tol.max()


def _check_neighbours(ref, tol):
    """A row or column off by one would move the values by far more than the bound."""
    t = np.max(tol) if np.ndim(tol) else tol
    if ref.shape[0] > 1:
        assert np.abs(ref[1:] - ref[:-1]).max() > 100 * t
    if ref.shape[1] > 1:
        assert np.abs(ref[:, 1:] - ref[:, :-1]).max() > 100 * t


@pytest.fixture(scope="module")
def cos_maps(ctx):
    """Integer X and integer W scaled by 2^-6 (three gathered maps of 100, 60 and 90 features): X W^T is exact in every operand
    mode (the fp16 copies only rescale by powers of two), so the argument of the cosine is fp32(z + b), one rounding."""
    rng = np.random.default_rng(41)
    n, d_in = 1000, 40
    X = rng.integers(-3, 4, (n, d_in)).astype(np.float64)
    Ws = [rng.integers(-3, 4, (m, d_in)) * 2.0 ** -6 for m in (100, 60, 90)]
    bs = [rng.random(m) * 2 * np.pi for m in (100, 60, 90)]
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in zip(Ws, bs)]
    return ctx.matrix(X.astype(np.float32)), X, rfs, np.concatenate(Ws, 0), np.concatenate(bs)


def _check_cosine_slab(ctx, x, handles, X, W, b, mode, row_begin, rows, c0, cols, shift, leak_measurable=True):
    out, lo, cs = _slab(ctx, x, handles, mode, row_begin, rows, c0, cols, shift)
    z = X[row_begin:row_begin + rows] @ W[c0:c0 + cols].T          # exact
    b32 = _f32(b[c0:c0 + cols])
    sh32 = _f32(shift) if shift is not None else np.zeros(cols)
    arg = _f32(z + b32)                                              # fmaf(acc, scale, bias): one rounding
    ref = np.cos(arg) - sh32
    # cosine error: Cody-Waite reduction + __cosf on [-pi, pi] (round_out = 0), or __cosf with its own range reduction
    # (~6e-8 |arg| of phase) in the rounded modes; then the fp32 subtraction of the shift
    cos_err = 2.0 ** -20 + (0.0 if SLAB_MODES[mode][1] == 0 else 2.5e-7 * np.abs(arg))
    tol = cos_err + 2.0 ** -23 + _output_tol(mode, ref)
    got = out + lo if lo is not None else out
    err = np.abs(got - ref)
    assert (err <= tol).all(), (mode, err.max(), np.unravel_index(np.argmax(err - tol), err.shape))
    _check_neighbours(ref, tol)
    _check_stored(mode, out, lo)
    if mode == "f16x2_pair":  # the pair must carry the unrounded fp32 slab of the same arithmetic to ~2^-22
        v, _, _ = _slab(ctx, x, handles, "f16x2", row_begin, rows, c0, cols, shift)
        assert (np.abs(got - v) <= 2.0 ** -22 * np.abs(v) + 2.0 ** -25).all()
    _check_colsums(cs, out + lo if lo is not None else out, np.cos(b32) - sh32, rows, leak_measurable)


# (maps, row_begin, rows, c0, cols): one map whole; a window that straddles all three gathered maps, with row_begin != 0 and
# rows % 32 != 0 (how the weighted solver calls it); a single element; all three maps whole
SLAB_WINDOWS = [(1, 0, 777, 0, 100), (3, 37, 913, 70, 130), (3, 500, 1, 160, 1), (3, 3, 250, 0, 250)]


@pytest.mark.parametrize("mode", list(SLAB_MODES))
@pytest.mark.parametrize("window", SLAB_WINDOWS, ids=lambda w: "maps%d_r%d+%d_c%d+%d" % w)
def test_projection_cosine(ctx, cos_maps, mode, window):
    x, X, rfs, W, b = cos_maps
    n_maps, row_begin, rows, c0, cols = window
    shift = np.random.default_rng(cols).uniform(-0.5, 0.5, cols)
    handles = [r.handle for r in rfs[:n_maps]]
    _check_cosine_slab(ctx, x, handles, X, W, b, mode, row_begin, rows, c0, cols, shift)


@pytest.mark.parametrize("dyn_tiles", [1, 0])
def test_projection_wraps_the_tile_ring(ctx, n_sms, dyn_tiles):
    """More than 8 tiles per CTA, with the tiles drawn from the counter (dyn_tiles 1) and strided statically (0).  The worst-case
    fp32 order error of ~4700 chunk sums per column is above what 50 leaked rows would add, so the leak is pinned by the smaller
    windows of test_projection_cosine."""
    rng = np.random.default_rng(43)
    d_in, cols = 40, 128
    rows = (9 * n_sms + 1) * TILE - 50
    X = rng.integers(-3, 4, (rows, d_in)).astype(np.float64)
    W = rng.integers(-3, 4, (cols, d_in)) * 2.0 ** -6
    b = rng.random(cols) * 2 * np.pi
    rf = ks.CosineRandomFeatures(ctx, W, b)
    x = ctx.matrix(X.astype(np.float32))
    ctx.set_option("dyn_tiles", dyn_tiles)
    try:
        _check_cosine_slab(ctx, x, [rf.handle], X, W, b, "tf32", 0, rows, 0, cols, np.full(cols, 0.25), leak_measurable=False)
    finally:
        ctx.set_option("dyn_tiles", 1)


@pytest.mark.parametrize("mode", list(SLAB_MODES))
def test_projection_rectified(ctx, mode):
    """KM_FLAG_RECT: RandomSignNode -> PaddedFFT -> LinearRectifier as one map; two gathered maps (different signs and alpha,
    one maxVal), a window across both.  The weights are cosines, so the reference is built from the operand the mode feeds the
    tensor core and the bound covers the fp32 accumulation; every output must be >= maxVal exactly.

    Split operands: X is not integer there (x + j 2^-12), so both cross products of the K-concatenated GEMM, x_lo w_hi and
    x_hi w_lo, carry data; the first two rows of the window are built so that each cross product of one entry adds up
    coherently, far above the bound."""
    rng = np.random.default_rng(44)
    n, d_in, max_val = 600, 100, 0.25
    row_begin, rows, c0, cols = 45, 517, 20, 70       # columns [20, 90) straddle the two 50-feature maps
    prec, _, _, proj_f16 = SLAB_MODES[mode]
    split = prec == KS_PRECISION_F16X2
    X = rng.integers(-3, 4, (n, d_in)).astype(np.float64)
    signs = [2.0 * rng.integers(0, 2, d_in) - 1.0 for _ in range(2)]
    alphas = [0.5, -1.0]
    P = ko.next_positive_power_of_two(d_in)
    f_idx, n_idx = np.arange(P // 2)[:, None], np.arange(d_in)[None, :]
    Wd = [s[None, :] * np.cos(2 * np.pi * ((f_idx * n_idx) % P) / P) for s in signs]   # the device's exact phase reduction
    for s, Wm in zip(signs, Wd):   # the dense map is PaddedFFT of the sign-flipped input
        assert np.abs(X @ Wm.T - ko.padded_fft(ko.random_sign_node(X, s))).max() < 1e-9
    W32 = _f32(np.concatenate(Wd, 0))
    if split:
        w_hi, w_lo = _split16(W32)
        c_star = c0 + 5
        X += rng.integers(-3, 4, X.shape) * 2.0 ** -12
        X[row_begin] = 3 * rng.choice([-1.0, 1.0], d_in) + 3 * 2.0 ** -12 * np.sign(w_hi[c_star])  # x_lo w_hi[c*] coherent
        X[row_begin + 1] = 3 * np.sign(w_lo[c_star])                                             # x_hi w_lo[c*] coherent
    x = ctx.matrix(X.astype(np.float32))
    assert np.array_equal(_f32(X), X)
    feats = [ks.LinearRectifier(max_val, al, ctx=ctx)(ks.PaddedFFT(ctx)(ks.RandomSignNode(s, ctx)(x))) for s, al in zip(signs, alphas)]
    handles = [f.rf_handles[0] for f in feats]
    if prec == KS_PRECISION_TF32 or (prec == KS_PRECISION_F16 and not proj_f16):
        Wop = round_tf32(W32).astype(np.float64)
    elif prec == KS_PRECISION_F16:
        Wop = W32.astype(np.float16).astype(np.float64)
    else:
        Wop = W32   # hi + lo: ~22 bits, the missing lo x lo product is inside the accumulation bound
    alpha = np.repeat(alphas, P // 2)
    out, lo, cs = _slab(ctx, x, handles, mode, row_begin, rows, c0, cols)
    Xw = X[row_begin:row_begin + rows]
    Wop, alpha = Wop[c0:c0 + cols], alpha[c0:c0 + cols]
    ref = np.maximum(max_val, Xw @ Wop.T - alpha)
    fft_ref = np.concatenate([ko.linear_rectifier(ko.padded_fft(ko.random_sign_node(Xw, s)), max_val, al)
                              for s, al in zip(signs, alphas)], 1)[:, c0:c0 + cols]
    mag = np.abs(Xw) @ np.abs(Wop).T
    # fp32 accumulation: <= 2^-23 |partial| per MMA step (13 tf32 / 7 fp16 / 19 split steps of K); the split mode also drops
    # x_lo w_lo (2^-22 |x||w|)
    tol = (2.0 ** -17 if split else 2.0 ** -16) * mag + EPS32 * (np.abs(ref) + 1) + _output_tol(mode, ref)
    got = out + lo if lo is not None else out
    err = np.abs(got - ref)
    assert (err <= tol).all(), (mode, err.max(), np.unravel_index(np.argmax(err - tol), err.shape))
    assert np.abs(got - fft_ref).max() < 2.0 ** -9 * mag.max()   # and the fp64 FFT, up to the operand rounding
    assert (out >= max_val).all() if lo is None else (got >= max_val).all()
    _check_neighbours(ref, tol)
    _check_stored(mode, out, lo)
    _check_colsums(cs, got if lo is None else out + lo, np.maximum(max_val, -alpha), rows)
    if split:   # dropping either cross product would move an entry far above the bound
        x_hi, x_lo = _split16(Xw)
        lh, hl = x_lo @ w_hi[c0:c0 + cols].T, x_hi @ w_lo[c0:c0 + cols].T
        assert (np.abs(lh) / tol).max() > 10 and (np.abs(hl) / tol).max() > 10, ((np.abs(lh) / tol).max(), (np.abs(hl) / tol).max())


def test_projection_rejects_slab_kinds_no_fit_requests(ctx, cos_maps):
    x, _, rfs, _, _ = cos_maps
    arr = (C.c_int64 * 1)(rfs[0].handle)
    out, lo = np.zeros((4, 4)), np.zeros((4, 4))
    for prec, round_out, pair in [(KS_PRECISION_TF32, 0, True), (KS_PRECISION_F16, 0, True), (KS_PRECISION_F16, 1, True),
                                  (KS_PRECISION_F16X2, 1, False), (7, 0, False)]:
        rc = lib().ks_debug_slab(ctx.handle, x.handle, arr, 1, prec, round_out, 0, 4, 0, 4, None, _ptr(out),
                                 _ptr(lo) if pair else None, 4, None)
        assert rc == KS_ERR_INVALID, (prec, round_out, pair)
    rc = lib().ks_debug_slab(ctx.handle, x.handle, arr, 1, KS_PRECISION_TF32, 0, 998, 4, 0, 4, None, _ptr(out), None, 4, None)
    assert rc == KS_ERR_INVALID   # window outside the rows


# ------------------------------------------------------------------------------------------ pooled Convolver (EPI_POOL)
# x_dim, y_dim, channels, conv size, pool stride, pool size, filters, images  ->  pools, patches per image
POOL_CASES = [
    (32, 32, 3, 6, 6, 8, 40, 3),     # 16 pools, 729 patches
    (32, 32, 3, 6, 13, 14, 33, 4),   # 4 pools (the CIFAR geometry), 729 patches
    (6, 9, 1, 3, 2, 2, 7, 11),       # 6 pools, 28 patches, non-square
    (8, 8, 1, 5, 4, 4, 64, 9),       # 1 pool, 16 patches
    (6, 10, 3, 3, 3, 4, 40, 7),      # 2 pools, exactly 32 patches, non-square
    (12, 7, 3, 5, 3, 2, 32, 10),     # 3 pools, 24 patches, non-square
    (14, 14, 1, 6, 3, 4, 40, 6),     # 9 pools, 81 patches
    (18, 6, 3, 3, 2, 2, 40, 5),      # 16 pools, 64 patches, non-square
]
RECTIFIERS = [(0.0, 0.5), (-1.5, 2.0), (2.5, -0.5), (0.0, 0.0)]   # (maxVal, alpha): integers and half-integers


def _pool_reference(imgs, filters, conv, max_val, alpha, stride, size, normalize=False, wmeans=None):
    return np.stack([ko.image_vectorizer(ko.pooler(ko.symmetric_rectifier(
        ko.convolve(im, filters, conv, normalize=normalize, whitener_means=wmeans), max_val, alpha), stride, size)) for im in imgs])


@pytest.mark.parametrize("precision", [KS_PRECISION_F16X2, KS_PRECISION_F16], ids=["parity", "f16"])
@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: "%dx%dx%d_conv%d_s%d_p%d_f%d_n%d" % c)
def test_pooled_convolver_is_exact(ctx, case, precision):
    """Pixels in [0, 15], integer filters in [-3, 3] (scaled to <= 4096 on the device): every patch product sum stays below
    2^23 and every pool sum of integers and half-integers below 2^22, so each fp32 sum and atomic is exact and the fused chain
    must equal the fp64 oracle bit for bit."""
    xd, yd, ch, conv, stride, size, nf, n = case
    rng = np.random.default_rng(xd * 1000 + yd * 10 + nf)
    imgs = rng.integers(0, 16, (n, xd, yd, ch)).astype(np.float64)
    filters = rng.integers(-3, 4, (nf, conv * conv * ch)).astype(np.float64)
    max_val, alpha = RECTIFIERS[POOL_CASES.index(case) % len(RECTIFIERS)]
    assert (conv * conv * ch) * 15 * 4096 < 2 ** 23
    conv_node = ks.Convolver(ctx, filters, xd, yd, ch, None, normalize_patches=False)
    chain = conv_node.andThen(ks.SymmetricRectifier(max_val, alpha)).andThen(ks.Pooler(stride, size)).andThen(ks.ImageVectorizer())
    ref = _pool_reference(imgs, filters, conv, max_val, alpha, stride, size)
    assert np.abs(ref).max() < 2 ** 22
    ctx.set_option("precision", precision)
    try:
        got = chain(ctx.matrix(ks.images_to_matrix(imgs))).to_numpy()
    finally:
        ctx.set_option("precision", KS_PRECISION_F16X2)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), (np.abs(got - ref).max(), np.unravel_index(np.argmax(np.abs(got - ref)), ref.shape))


def test_pooled_convolver_normalized_with_whitener_means(ctx):
    """Normalised patches and whitener means on the non-square 16-pool geometry, gated like the CIFAR featurizer test of
    test_gpu_parity.py."""
    rng = np.random.default_rng(45)
    xd, yd, ch, conv, stride, size, nf, n = 18, 6, 3, 3, 2, 2, 40, 8
    imgs = rng.integers(0, 256, (n, xd, yd, ch)).astype(np.float64)
    filters = rng.standard_normal((nf, conv * conv * ch)) / 10.0
    wmeans = rng.standard_normal(conv * conv * ch) * 0.05
    conv_node = ks.Convolver(ctx, filters, xd, yd, ch, wmeans, normalize_patches=True, var_constant=10.0)
    chain = conv_node.andThen(ks.SymmetricRectifier(alpha=0.25)).andThen(ks.Pooler(stride, size)).andThen(ks.ImageVectorizer())
    ref = _pool_reference(imgs, filters, conv, 0.0, 0.25, stride, size, normalize=True, wmeans=wmeans)
    got = chain(ctx.matrix(ks.images_to_matrix(imgs))).to_numpy()
    assert np.abs(got - ref).max() < 1e-4 * np.abs(ref).max(), np.abs(got - ref).max() / np.abs(ref).max()
    ctx.set_option("precision", KS_PRECISION_F16)
    try:
        fast = chain(ctx.matrix(ks.images_to_matrix(imgs))).to_numpy()
    finally:
        ctx.set_option("precision", KS_PRECISION_F16X2)
    assert np.abs(fast - ref).max() < 5e-3 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------ fit arrangements on one GPU
OPTION_DEFAULTS = {"lookahead": 0, "dyn_tiles": 1, "proj_f16": 1, "custom_solve": -1}
# options -> the look-ahead the fit reports (NBUF = lookahead + 2 slab buffers rotate)
ARRANGEMENTS = [
    ({"lookahead": 1}, 1), ({"lookahead": 2}, 2), ({"lookahead": 4}, 4),
    ({"dyn_tiles": 0}, 1), ({"proj_f16": 0}, 1), ({"custom_solve": 1}, 1),
]


@pytest.fixture(scope="module")
def fit_problem(ctx):
    """Three gathered cosine maps (768 features) in blocks of 112: 7 blocks, so every one of the LA + 2 buffers is reused."""
    rng = np.random.default_rng(46)
    n, d_in, n_out, k, bs = 3000, 44, 256, 10, 112
    X = rng.standard_normal((n, d_in))
    cls = rng.integers(0, k, n)
    params = [ko.cosine_random_features_params(d_in, n_out, 0.17, rng) for _ in range(3)]
    x = ctx.matrix(X.astype(np.float32))
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
    Xd = X.astype(np.float32).astype(np.float64)
    F = np.concatenate([ko.cosine_random_features(Xd, W, b) for W, b in params], 1)
    Y = ko.class_label_indicators(cls, k)
    refs = {iters: np.concatenate(ko.block_ls_fit(F, Y, bs, iters, 2.0)[0], 0) for iters in (1, 2)}
    return feats, ctx.labels_from_classes(cls, k), bs, refs, rfs


@pytest.mark.parametrize("options,lookahead", ARRANGEMENTS, ids=lambda v: str(v).replace(" ", "") if isinstance(v, dict) else None)
def test_fit_arrangements(ctx, fit_problem, options, lookahead):
    feats, y, bs, refs, _ = fit_problem
    fast = options.get("proj_f16") == 0
    try:
        for name, value in options.items():
            ctx.set_option(name, value)
        for iters in (1, 2):   # one sweep, and two with the factors cached
            model = ks.BlockLeastSquaresEstimator(bs, iters, 2.0, precision="f16" if fast else "default").fit(feats, y)
            stats = ctx.last_fit_stats()
            assert stats["num_blocks"] == 7
            assert stats["lookahead"] == lookahead and stats["mma"] == ("f16" if fast else "f16x2")
            if options.get("custom_solve") == 1:
                assert stats["solve"].startswith("dmma-kernel")
            W = np.concatenate(model.xs, 0)
            rel = np.linalg.norm(W - refs[iters]) / np.linalg.norm(refs[iters])
            assert rel < (W_TOL_FAST if fast else W_TOL), (iters, rel)
    finally:
        for name, value in OPTION_DEFAULTS.items():
            ctx.set_option(name, value)


def test_removed_fit_options_rejected(ctx):
    """The fit has one stream arrangement and always times its phases: the options that selected otherwise are unknown."""
    for name in ("pipeline", "timing"):
        with pytest.raises(ks.KeystoneError):
            ctx.set_option(name, 1)
