"""Each step of BlockLeastSquaresEstimator.fit (engine.cu::fit_blockls) against fp64, from the state the fit itself held:
ks_debug_blockls_capture copies the shift, delta, the exact diagonal, H, rhs, dW, the slab planes and the residual before and
after chosen steps (sweep, block) of one fit, and tests/blockls_steps_ref.py restates each step in fp64 with an entrywise bound
derived from the device's arithmetic.

The problems make the shift-then-correct terms real: generated features take their shift from the first `sample_rows` = 257
rows, so delta (and with it N delta delta^T and the update's constant delta^T dW) is far above rounding; N = 6001 is not a
multiple of the 128-row tile; the last block is ragged and not a multiple of 32; there are more blocks than the LA + 2 rotating
buffers; k = 1100 > 8 * 132 routes the DMMA solve to chol_solve_kernel<16>.  Every operand mode the fit selects is covered:
fp16 pairs (parity) and fp16 (fast) on cosine features, tf32 pairs (parity) and tf32 on materialised features, tf32 pairs on
rectified PaddedFFT features.

Terms the captured state cannot pin: -delta rsum^T in build_rhs_kernel is at rounding size in every fit (the residual stays
centred, so rsum ~ 0), and no device test pins it (tests/test_blockls_steps_algebra.py only shows that rhs_bound would reject its
absence for a residual that is not centred); the dropped lo * lo products and the cross terms of the pairs are below the
accumulation bound on random data (pinned exactly by tests/test_gpu_split_gram.py, tests/test_gpu_split_pairs.py and
tests/test_gpu_kmajor.py).

test_real_geometry runs the same checks at the benchmark's shapes (C3 maps, b = 4096, k = 1000), and compares the captured slab
with the oracle's fp64 cosines; test_two_rank_capture (2 GPUs) checks that the ranks assemble and solve bit-identical systems.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import KS_PRECISION_F16, KS_PRECISION_F16X2, check, lib
from keystone_b200.context import feature_source_args
from oracle import keystone_oracle as ko

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import blockls_steps_ref as st  # noqa: E402

pytestmark = pytest.mark.gpu

W_TOL = 1e-4        # parity mode (tests/test_gpu_parity.py)
W_TOL_FAST = 1.5e-3  # 10-bit operand modes
SHIFT, DELTA, DIAG, H, RHS, DW, SLAB_HI, SLAB_LO, R_BEFORE, R_AFTER, SCALES, COUNT = range(12)
N, BS, LAM = 6001, 128, 200.0   # lambda W_old 20x above the rhs bound (at lambda = 50 it was 6-8x)
KS_ERR_INVALID = -1


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


class Options:
    """Sets context options and restores the library defaults on exit."""
    DEFAULTS = {"sample_rows": 16384, "lookahead": 0, "custom_solve": -1}

    def __init__(self, ctx, **kw):
        self.ctx, self.kw = ctx, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.ctx.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            self.ctx.set_option(k, self.DEFAULTS[k])


# ------------------------------------------------------------------------------------------------------ problems
def _f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def problem(ctx, source, k, seed):
    """(data, F fp64 as the device sees it, classes)."""
    rng = np.random.default_rng(seed)
    cls = rng.integers(0, k, N)
    if source == "cos":   # two maps of 470 + 471 features: D = 941, blocks of 128, the last one 45 wide
        X = (0.5 * rng.standard_normal((k, 30))[cls] + rng.standard_normal((N, 30))).astype(np.float32)
        params = [ko.cosine_random_features_params(30, m, 0.2, rng) for m in (470, 471)]
        params = [(_f32(W), _f32(b)) for W, b in params]
        rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
        x = ctx.matrix(X)
        data = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
        F = np.concatenate([ko.cosine_random_features(X.astype(np.float64), W, b) for W, b in params], 1)
        return data, F, cls
    if source == "fft":   # two rectified PaddedFFT branches of 784 inputs: D = 1024, cut to 1005 by num_features
        X = rng.random((N, 784)).astype(np.float32)
        signs = [2.0 * rng.integers(0, 2, 784) - 1.0 for _ in range(2)]
        branches = [ks.RandomSignNode(s, ctx).andThen(ks.PaddedFFT(ctx)).andThen(ks.LinearRectifier(0.0, ctx=ctx)) for s in signs]
        data = ks.Pipeline.gather(branches).andThen(ks.VectorCombiner())(ctx.matrix(X))
        return data, data.to_numpy(), cls
    F = (rng.standard_normal((N, 941)) + 0.5 * rng.standard_normal((k, 941))[cls] + 2.0).astype(np.float32)
    return ctx.matrix(F), F.astype(np.float64), cls


# id: (source, precision, mma, k, sweeps, lookahead, custom_solve, num_features)
CASES = {
    "cos-parity-k10": ("cos", "f16x2", "f16x2", 10, 3, 1, 0, None),
    "cos-parity-k1100": ("cos", "f16x2", "f16x2", 1100, 1, 4, 1, None),
    "cos-fast-k10": ("cos", "f16", "f16", 10, 3, 4, 1, None),
    "mat-parity-k10": ("mat", "default", "tf32x2", 10, 3, 4, 0, None),
    "mat-tf32-k1100": ("mat", "tf32", "tf32x1", 1100, 1, 1, 1, None),
    "fft-parity-k10": ("fft", "default", "tf32x2", 10, 3, 1, 1, 1005),
}


def capture_fit(ctx, fit, steps, widths, n, k, what):
    """Arms `steps` ((sweep, block) pairs) with buffers for the entries in `what`, runs fit(), returns {step: {entry: array}}."""
    sizes = {SHIFT: lambda b: b, DELTA: lambda b: b, DIAG: lambda b: b, H: lambda b: b * b, RHS: lambda b: b * k,
             DW: lambda b: b * k, SLAB_HI: lambda b: n * b, SLAB_LO: lambda b: n * b, R_BEFORE: lambda b: n * k,
             R_AFTER: lambda b: n * k, SCALES: lambda b: 4}
    out = {}
    for s, j in steps:
        bufs = {e: np.full(sizes[e](widths[j]), np.nan) for e in what if not (s > 0 and e in (H, DIAG))}
        arr = (C.c_void_p * COUNT)(*[bufs[e].ctypes.data if e in bufs else None for e in range(COUNT)])
        check(ctx.handle, lib().ks_debug_blockls_capture(ctx.handle, s, j, arr))
        out[(s, j)] = bufs
    model = fit()
    for (s, j), bufs in out.items():
        b = widths[j]
        for e, v in bufs.items():
            assert not np.isnan(v).any(), f"step {(s, j)} entry {e} not captured"
        shaped = {e: v.reshape(b, b, order="F") if e == H else v.reshape(k, b).T if e in (RHS, DW)
                  else v.reshape(n, -1) if e in (SLAB_HI, SLAB_LO, R_BEFORE, R_AFTER) else v for e, v in bufs.items()}
        out[(s, j)] = shaped
    return model, out


def guard(name, term, bound, margin):
    """A term the check guards is far above its bound: dropping it would exceed the bound `margin` times over somewhere."""
    r = st.ratio(term, bound)
    assert r > margin, (name, r)


def projection_planes(ctx, data, mma, s0, e0, shift):
    """The planes of feature columns [s0, e0) from the projection alone (ks_debug_slab) with the fit's shift: fp16 pairs, the
    fp16 slab, or the unrounded fp32 slab split into tf32 pairs as center_round_kernel splits it (shift already applied)."""
    _, x, rfs, n_rfs = feature_source_args(data)
    cols = e0 - s0
    dh, dl = np.zeros((N, cols)), np.zeros((N, cols))
    prec, round_out, lo = {"f16x2": (KS_PRECISION_F16X2, 0, dl), "f16": (KS_PRECISION_F16, 1, None),
                           "tf32x2": (KS_PRECISION_F16X2, 0, None)}[mma]
    check(ctx.handle, lib().ks_debug_slab(ctx.handle, x, rfs, n_rfs, prec, round_out, 0, N, s0, cols,
                                          np.ascontiguousarray(shift).ctypes.data_as(C.c_void_p), dh.ctypes.data_as(C.c_void_p),
                                          None if lo is None else lo.ctypes.data_as(C.c_void_p), cols, None))
    if mma == "tf32x2":
        return st.center_round(dh, np.zeros(cols), True)
    return dh, dl


def _report(name, err, bound, worst):
    r = st.ratio(err, bound)
    worst[name] = max(worst.get(name, 0.0), r)
    assert r <= 1.0, (name, r)


@pytest.mark.parametrize("case", list(CASES))
def test_fit_steps_against_fp64(ctx, case):
    source, precision, mma, k, sweeps, la, cs, nf = CASES[case]
    data, F, cls = problem(ctx, source, k, seed=len(case) + k)
    D = nf or F.shape[1]
    bounds = ko.block_bounds(D, BS)
    nb = len(bounds)
    widths = [e - s for s, e in bounds]
    assert N % 128 and widths[-1] % 32 and nb > la + 2
    y = ctx.labels_from_classes(cls, k)
    Y = ko.class_label_indicators(cls, k)
    est = ks.BlockLeastSquaresEstimator(BS, sweeps, LAM, nf, precision=precision)
    blocks = sorted({0, 1, nb - 1})
    steps = [(s, j) for s in range(sweeps) for j in blocks]
    pair = st.MODES[mma][0]
    what = [SHIFT, DELTA, H, RHS, DW, SLAB_HI, SLAB_LO, R_BEFORE, R_AFTER, SCALES] + ([DIAG] if pair else [])
    generated = source != "mat"
    with Options(ctx, sample_rows=257 if generated else 16384, lookahead=la, custom_solve=cs):
        est.fit(data, y)
        plain = ctx.last_fit_stats()
        model, cap = capture_fit(ctx, lambda: est.fit(data, y), steps, widths, N, k, what)
        stats = ctx.last_fit_stats()
    assert stats["mma"] == mma and stats["lookahead"] == la
    assert stats["solve"] == ("dmma-kernel" if cs else "potrs")
    # the library's own count of the kernels it enqueues: a launch added under a capture without its count would not show here,
    # which is why the capture converts on the host and enqueues nothing but copies
    assert stats["launches"] == plain["launches"], "arming a capture changed what the fit launches"
    chain = stats["chain_rows"]
    means = model.feature_means
    xs = model.xs
    worst = {}
    # identities: the residual chain, the slabs across sweeps, the model
    R0 = _f32(Y - model.b_opt)
    assert np.array_equal(cap[(0, 0)][R_BEFORE], R0)
    order = [(s, j) for s in range(sweeps) for j in range(nb)]
    for t in range(len(order) - 1):
        if order[t] in cap and order[t + 1] in cap:
            assert np.array_equal(cap[order[t + 1]][R_BEFORE], cap[order[t]][R_AFTER]), (order[t], order[t + 1])
    for j in blocks:
        for s in range(1, sweeps):
            for e in (SHIFT, DELTA, SLAB_HI, SLAB_LO):
                assert np.array_equal(cap[(s, j)][e], cap[(0, j)][e]), (s, j, e)
        c0 = cap[(0, j)]
        assert np.array_equal(means[j], c0[SHIFT] + c0[DELTA])
        Wsum = np.zeros_like(c0[DW])
        for s in range(sweeps):
            Wsum = Wsum + cap[(s, j)][DW]
        assert np.array_equal(xs[j], Wsum)
        hi, lo = c0[SLAB_HI], c0[SLAB_LO]
        s0, e0 = bounds[j]
        if source == "mat":   # center_round_kernel on the fp32 features with the exact column mean
            assert np.abs(c0[SHIFT] - F[:, s0:e0].mean(0)).max() <= 2.0 ** -23 * np.abs(F[:, s0:e0]).max()
            rh, rl = st.center_round(F[:, s0:e0], c0[SHIFT], pair)
            assert np.array_equal(hi, rh) and np.array_equal(lo, rl)
        else:   # the projection alone (ks_debug_slab), with the captured shift, gives the same planes
            dh, dl = projection_planes(ctx, data, mma, s0, e0, c0[SHIFT])
            assert np.array_equal(hi, dh) and np.array_equal(lo, dl)
        if source == "cos":
            # the shift is the mean of the first sample rows, to the fp32 sums and the cosine's error
            # (the fast mode estimates it from fp16 slabs: 2^-12 relative per value)
            assert np.abs(c0[SHIFT] - F[:257, s0:e0].mean(0)).max() < (1e-5 if pair else 2.0 ** -11)
        # fp64 references
        S = hi + lo
        delta = c0[DELTA]
        _report("delta", np.abs(delta - S.mean(0)), st.delta_bound(hi, lo), worst)
        if generated:   # a real shift correction: delta far above its bound
            guard("delta", np.abs(delta), st.delta_bound(hi, lo), 100)
        if pair:
            _report("diag", np.abs(c0[DIAG] - (S ** 2).sum(0)), st.diag_bound(hi, lo), worst)
            ssq = (S ** 2).sum(0)   # one fp32 ulp of the diagonal is far outside (rectified features may have zero columns)
            assert (2.0 ** -24 * ssq[ssq > 0] > 100 * st.diag_bound(hi, lo)[ssq > 0]).all()
        Hd = c0[H]
        Href = st.system(hi, lo, delta, LAM)
        bH = st.system_bound(hi, lo, delta, LAM, mma, chain)
        _report("H", np.abs(Hd - Href), bH, worst)
        if pair:
            _report("H diag", np.abs(np.diag(Hd) - (c0[DIAG] - N * delta ** 2 + LAM)),
                    4 * st.EPS64 * (c0[DIAG] + N * delta ** 2 + LAM), worst)
        if generated:
            guard("N delta delta^T", N * np.abs(np.outer(delta, delta)), bH, 10)
        assert (LAM > 10 * np.diag(bH)).all(), ("lambda", (np.diag(bH) / LAM).max())
        rs, ws = 1.0, 1.0
        W_old = None
        for s in range(sweeps):
            cs_ = cap[(s, j)]
            if mma in ("f16x2", "f16"):
                rs, ws = cs_[SCALES][0], cs_[SCALES][2]
            else:
                assert np.array_equal(cs_[SCALES], np.ones(4))
            R = cs_[R_BEFORE]
            rhs_ref = st.rhs_of(hi, lo, delta, R, LAM, W_old)
            bR = st.rhs_bound(hi, lo, delta, R, LAM, W_old, mma, chain, rs)
            _report("rhs", np.abs(cs_[RHS] - rhs_ref), bR, worst)
            if W_old is not None:
                guard("lambda W_old", LAM * np.abs(W_old), bR, 10)
            dW = cs_[DW]
            _report("solve", np.abs(Hd @ dW - cs_[RHS]), st.solve_bound(Hd, dW), worst)
            assert st.solve_bound(Hd, dW).max() < 1e-6 * np.abs(cs_[RHS]).max()
            upd_ref = st.update_of(hi, lo, delta, R, dW)
            bU = st.update_bound(hi, lo, delta, R, dW, mma, ws)
            _report("R_after", np.abs(cs_[R_AFTER] - upd_ref), bU, worst)
            if generated:
                guard("delta^T dW", np.abs(delta @ dW), bU.max(0), 10)
            W_old = dW if W_old is None else W_old + dW
    W = np.concatenate(xs, 0)
    ref, _, _ = ko.block_ls_fit(F, Y, BS, sweeps, LAM, num_features=nf)
    rel = np.linalg.norm(W - np.concatenate(ref, 0)) / np.linalg.norm(np.concatenate(ref, 0))
    print(f"{case}: chain {chain}, rel-Fro(W) {rel:.3e}; largest error / bound: "
          + ", ".join(f"{n_} {r:.3g}" for n_, r in worst.items()))
    assert rel < (W_TOL if pair else W_TOL_FAST)


def test_linear_map_estimator_steps(ctx):
    """ks_linear_map_fit is one block, one sweep of the same fit: its slab, delta, system, rhs and solve through the capture."""
    rng = np.random.default_rng(5)
    n, d, k, lam = 3001, 77, 6, 2.0
    F = (rng.standard_normal((n, d)) + 1.5).astype(np.float32)
    Yv = rng.standard_normal((n, k)).astype(np.float32)
    bufs = {e: np.full(sz, np.nan) for e, sz in ((SHIFT, d), (DELTA, d), (DIAG, d), (H, d * d), (RHS, d * k), (DW, d * k),
                                                  (SLAB_HI, n * d), (SLAB_LO, n * d), (R_BEFORE, n * k))}
    arr = (C.c_void_p * COUNT)(*[bufs[e].ctypes.data if e in bufs else None for e in range(COUNT)])
    check(ctx.handle, lib().ks_debug_blockls_capture(ctx.handle, 0, 0, arr))
    m = ks.LinearMapEstimator(lam).fit(ctx.matrix(F), ctx.matrix(Yv))
    stats = ctx.last_fit_stats()
    assert stats["mma"] == "tf32x2"
    assert not any(np.isnan(v).any() for v in bufs.values())
    hi, lo = bufs[SLAB_HI].reshape(n, d), bufs[SLAB_LO].reshape(n, d)
    rh, rl = st.center_round(F.astype(np.float64), bufs[SHIFT], True)
    assert np.array_equal(hi, rh) and np.array_equal(lo, rl)
    delta, chain = bufs[DELTA], stats["chain_rows"]
    assert st.ratio(np.abs(delta - (hi + lo).mean(0)), st.delta_bound(hi, lo)) <= 1
    assert st.ratio(np.abs(bufs[DIAG] - ((hi + lo) ** 2).sum(0)), st.diag_bound(hi, lo)) <= 1
    Hd = bufs[H].reshape(d, d, order="F")
    assert st.ratio(np.abs(Hd - st.system(hi, lo, delta, lam)), st.system_bound(hi, lo, delta, lam, "tf32x2", chain)) <= 1
    R = bufs[R_BEFORE].reshape(n, k)
    assert np.array_equal(R, _f32(Yv.astype(np.float64) - m.b_opt))
    rhs = bufs[RHS].reshape(k, d).T
    assert st.ratio(np.abs(rhs - st.rhs_of(hi, lo, delta, R, lam, None)), st.rhs_bound(hi, lo, delta, R, lam, None, "tf32x2", chain, 1.0)) <= 1
    dW = bufs[DW].reshape(k, d).T
    assert st.ratio(np.abs(Hd @ dW - rhs), st.solve_bound(Hd, dW)) <= 1
    assert np.array_equal(m.xs[0], dW)
    assert np.array_equal(m.feature_means[0], bufs[SHIFT] + delta)


def test_capture_requests_and_disarming(ctx):
    h = np.zeros(16)
    arr = (C.c_void_p * COUNT)(*[h.ctypes.data if e == H else None for e in range(COUNT)])
    assert lib().ks_debug_blockls_capture(ctx.handle, 1, 0, arr) == KS_ERR_INVALID
    arr = (C.c_void_p * COUNT)(*[h.ctypes.data if e == DIAG else None for e in range(COUNT)])
    assert lib().ks_debug_blockls_capture(ctx.handle, 2, 0, arr) == KS_ERR_INVALID
    F = np.random.default_rng(1).standard_normal((300, 16))
    arr = (C.c_void_p * COUNT)(*[h.ctypes.data if e == SHIFT else None for e in range(COUNT)])
    # a request for a step the fit does not have writes nothing
    check(ctx.handle, lib().ks_debug_blockls_capture(ctx.handle, 5, 7, arr))
    ks.BlockLeastSquaresEstimator(8, 1, 1.0).fit(ctx.matrix(F), ctx.matrix(F[:, :2]))
    assert not h.any()
    # a fit that throws still takes the request: the next good fit is not armed
    check(ctx.handle, lib().ks_debug_blockls_capture(ctx.handle, 0, 0, arr))
    with pytest.raises(ks.KeystoneError):
        ks.BlockLeastSquaresEstimator(8, 1, 1.0).fit(ctx.matrix(F), ctx.matrix(F[:299, :2]))
    ks.BlockLeastSquaresEstimator(8, 1, 1.0).fit(ctx.matrix(F), ctx.matrix(F[:, :2]))
    assert not h.any()
    # an armed good fit does write the shift (8 of the 16 values: the block width)
    check(ctx.handle, lib().ks_debug_blockls_capture(ctx.handle, 0, 0, arr))
    ks.BlockLeastSquaresEstimator(8, 1, 1.0).fit(ctx.matrix(F), ctx.matrix(F[:, :2]))
    assert h[:8].any() and not h[8:].any()


# ------------------------------------------------------------------------------------------------------ real geometry
def test_real_geometry(ctx):
    """The benchmark's configuration in miniature: C3 cosine maps (440 -> 4096, gamma 0.0555; 4 of the 16), k = 1000, b = 4096,
    lambda = 1, N = 8192, shift from 2048 sample rows; blocks 0 and 3 of the parity-mode fit, whose Gram chains are 4096 rows
    long.  The steps are checked against the captured slab as above, and the captured slab against the oracle's fp64 cosines:
    H and rhs built from those cosines differ from the device's by at most the bound plus the slab's measured feature error."""
    rng = np.random.default_rng(2)
    n, d_in, b, k, lam = 8192, 440, 4096, 1000, 1.0
    params = [(_f32(rng.standard_normal((b, d_in)) * 0.0555), _f32(rng.random(b) * 2 * np.pi)) for _ in range(4)]
    X = rng.standard_normal((n, d_in), dtype=np.float32)
    wstar = rng.standard_normal((16, k)).astype(np.float32)
    cls = np.argmax(X[:, :16] @ wstar + 0.1 * rng.standard_normal((n, k)).astype(np.float32), axis=1)
    rfs = [ks.CosineRandomFeatures(ctx, W, bb) for W, bb in params]
    data = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(ctx.matrix(X))
    y = ctx.labels_from_classes(cls, k)
    what = [SHIFT, DELTA, DIAG, H, RHS, DW, SLAB_HI, SLAB_LO, R_BEFORE, SCALES]
    with Options(ctx, sample_rows=2048):
        model, cap = capture_fit(ctx, lambda: ks.BlockLeastSquaresEstimator(b, 1, lam).fit(data, y), [(0, 0), (0, 3)], [b] * 4, n, k,
                                 what)
    stats = ctx.last_fit_stats()
    assert stats["mma"] == "f16x2"
    chain = stats["chain_rows"]
    X64 = X.astype(np.float64)
    worst = {}
    for j in (0, 3):
        c = cap[(0, j)]
        hi, lo, delta, Hd, R, rhs, dW = c[SLAB_HI], c[SLAB_LO], c[DELTA], c[H], c[R_BEFORE], c[RHS], c[DW]
        S = hi + lo
        _report("delta", np.abs(delta - S.mean(0)), st.delta_bound(hi, lo), worst)
        _report("diag", np.abs(c[DIAG] - (S ** 2).sum(0)), st.diag_bound(hi, lo), worst)
        bH = st.system_bound(hi, lo, delta, lam, "f16x2", chain)
        _report("H", np.abs(Hd - st.system(hi, lo, delta, lam)), bH, worst)
        bR = st.rhs_bound(hi, lo, delta, R, lam, None, "f16x2", chain, c[SCALES][0])
        _report("rhs", np.abs(rhs - st.rhs_of(hi, lo, delta, R, lam, None)), bR, worst)
        _report("solve", np.abs(Hd @ dW - rhs), st.solve_bound(Hd, dW), worst)
        assert np.array_equal(model.xs[j], dW)
        # against the oracle's cosines: |S_hat - S| <= e entrywise moves S^T S by e (|S|^T 1 + 1^T |S| + N e) and S^T R by e 1^T |R|
        Sref = ko.cosine_random_features(X64, *params[j]) - c[SHIFT]
        err = np.abs(S - Sref)
        e = float(err.max())
        worst["feature error"] = e
        # feature error: the cosine (2^-20 absolute), the shift subtraction and the pair (2^-23, 2^-22 |S|), and the projection
        # X W^T on split fp16 operands concatenated along K (3 d_in deep: one fp32 ulp per 8-deep group of the partial sum, the
        # dropped lo * lo, the fp32 bias add), which moves the cosine's argument by up to that much
        W, bb = params[j]
        proj = np.abs(X64) @ np.abs(W).T
        arg_err = (-(-3 * d_in // 8) * 2.0 ** -23 + 2.0 ** -21) * proj + 2.0 ** -24 * (proj + np.abs(bb))
        _report("features vs oracle cosines", err, 2.0 ** -20 + 2.0 ** -23 + 2.0 ** -22 * np.abs(Sref) + 2.0 ** -25 + arg_err, worst)
        col = np.abs(Sref).sum(0)
        _report("H vs oracle cosines", np.abs(Hd - st.system(Sref, 0 * Sref, delta, lam)),
                bH + e * (col[:, None] + col[None, :] + n * e), worst)
        _report("rhs vs oracle cosines", np.abs(rhs - st.rhs_of(Sref, 0 * Sref, delta, R, lam, None)),
                bR + e * np.abs(R).sum(0)[None, :], worst)
    print("real geometry (N 8192, b 4096, k 1000): " + ", ".join(f"{n_} {r:.3g}" for n_, r in worst.items()))


# ------------------------------------------------------------------------------------------------------ two ranks
def _two_rank_worker(rank, world, id_holder, ret):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import keystone_b200 as ks
    from keystone_b200._capi import check, lib
    from oracle import keystone_oracle as ko
    rng = np.random.default_rng(31)
    n, d_in, k = 6001, 30, 10
    X = rng.standard_normal((n, d_in)).astype(np.float32)
    cls = rng.integers(0, k, n)
    params = [ko.cosine_random_features_params(d_in, m, 0.2, rng) for m in (470, 471)]
    lo, hi = ks.shard_range(n, rank, world)
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    ctx.set_option("sample_rows", 257)
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    data = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(ctx.matrix(X[lo:hi]))
    nl = hi - lo
    widths = [e - s for s, e in ko.block_bounds(941, BS)]
    steps = [(0, 0), (0, 1), (1, 0)]
    sizes = {SHIFT: lambda b: b, DELTA: lambda b: b, DIAG: lambda b: b, H: lambda b: b * b, RHS: lambda b: b * k,
             DW: lambda b: b * k, SLAB_HI: lambda b: nl * b, SLAB_LO: lambda b: nl * b, R_BEFORE: lambda b: nl * k,
             R_AFTER: lambda b: nl * k}
    bufs = {}
    for s, j in steps:   # every rank arms the same steps (the copies block the host between collectives)
        bufs[(s, j)] = {e: np.full(f(widths[j]), np.nan) for e, f in sizes.items() if not (s > 0 and e in (H, DIAG))}
        arr = (C.c_void_p * COUNT)(*[bufs[(s, j)][e].ctypes.data if e in bufs[(s, j)] else None for e in range(COUNT)])
        check(ctx.handle, lib().ks_debug_blockls_capture(ctx.handle, s, j, arr))
    ks.BlockLeastSquaresEstimator(BS, 2, LAM).fit(data, ctx.labels_from_classes(cls[lo:hi], k))
    ret[f"stats{rank}"] = ctx.last_fit_stats()
    ret[f"cap{rank}"] = bufs
    ctx.close()


def test_two_rank_capture():
    """Rows sharded over two ranks: H, rhs and dW are bitwise equal across the ranks (G and C are all-reduced, the solves sharded
    by columns and broadcast), and the steps pass the checks above with each rank's rows (the system over both ranks' slabs,
    the update with each rank's own rows)."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mgr = mp.Manager()
    id_holder, ret = mgr.dict(), mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_two_rank_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    c0, c1 = ret["cap0"], ret["cap1"]
    stats = ret["stats0"]
    assert stats["mma"] == "f16x2" and stats["world"] == 2
    k, chain = 10, stats["chain_rows"]
    for step in c0:
        for e in (H, RHS, DW, DELTA, SHIFT, DIAG):
            if e in c0[step]:
                assert not np.isnan(c0[step][e]).any() and np.array_equal(c0[step][e], c1[step][e]), (step, e)
    for j in (0, 1):
        b = c0[(0, j)][SHIFT].size
        planes = [(c[(0, j)][SLAB_HI].reshape(-1, b), c[(0, j)][SLAB_LO].reshape(-1, b)) for c in (c0, c1)]
        hi = np.concatenate([p[0] for p in planes])
        lo = np.concatenate([p[1] for p in planes])
        delta = c0[(0, j)][DELTA]
        Hd = c0[(0, j)][H].reshape(b, b, order="F")
        assert st.ratio(np.abs(delta - (hi + lo).mean(0)), st.delta_bound(hi, lo)) <= 1
        assert st.ratio(np.abs(Hd - st.system(hi, lo, delta, LAM)), st.system_bound(hi, lo, delta, LAM, "f16x2", chain)) <= 1
        R = np.concatenate([c[(0, j)][R_BEFORE].reshape(-1, k) for c in (c0, c1)])
        rhs = c0[(0, j)][RHS].reshape(k, b).T
        dW = c0[(0, j)][DW].reshape(k, b).T
        assert st.ratio(np.abs(rhs - st.rhs_of(hi, lo, delta, R, LAM, None)),
                        st.rhs_bound(hi, lo, delta, R, LAM, None, "f16x2", chain, 1.0)) <= 1
        assert st.ratio(np.abs(Hd @ dW - rhs), st.solve_bound(Hd, dW)) <= 1
        for c, (h, l) in zip((c0, c1), planes):   # each rank's rows updated with its own slab
            Rb, Ra = c[(0, j)][R_BEFORE].reshape(-1, k), c[(0, j)][R_AFTER].reshape(-1, k)
            assert st.ratio(np.abs(Ra - st.update_of(h, l, delta, Rb, dW)), st.update_bound(h, l, delta, Rb, dW, "f16x2", 1.0)) <= 1
        for c in (c0, c1):   # the residual chain, step (0, 0) -> (0, 1), and the regenerated slab of sweep 1, on each rank
            assert np.array_equal(c[(0, 1)][R_BEFORE], c[(0, 0)][R_AFTER])
            assert np.array_equal(c[(1, 0)][SLAB_HI], c[(0, 0)][SLAB_HI]) and np.array_equal(c[(1, 0)][SLAB_LO], c[(0, 0)][SLAB_LO])


# ------------------------------------------------------------------------------------------------------ row order
@pytest.mark.parametrize("sweeps", [1, 2])
@pytest.mark.parametrize("precision", ["f16x2", "f16"])
@pytest.mark.parametrize("order", ["sorted", "shuffled"])
def test_row_order_against_the_oracle(ctx, order, precision, sweeps):
    """Rows delivered sorted by class (as directory-based loaders do) make the first sample rows unrepresentative: the shift is far
    from the mean and delta is large.  The fit must still meet the library's gates against the fp64 oracle."""
    rng = np.random.default_rng(77)
    n, k, d_in = 16000, 10, 40
    cls = rng.integers(0, k, n)
    if order == "sorted":
        cls = np.sort(cls)
    X = (1.0 * rng.standard_normal((k, d_in))[cls] + rng.standard_normal((n, d_in))).astype(np.float32)
    params = [(_f32(W), _f32(b)) for W, b in (ko.cosine_random_features_params(d_in, 256, 0.3, rng) for _ in range(2))]
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    data = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(ctx.matrix(X))
    F = np.concatenate([ko.cosine_random_features(X.astype(np.float64), W, b) for W, b in params], 1)
    Y = ko.class_label_indicators(cls, k)
    with Options(ctx, sample_rows=1024):
        model = ks.BlockLeastSquaresEstimator(256, sweeps, 1.0, precision=precision).fit(data, ctx.labels_from_classes(cls, k))
    xs, _, mus = ko.block_ls_fit(F, Y, 256, sweeps, 1.0)
    shift_gap = max(np.abs(F[:1024, s:e].mean(0) - m).max() for (s, e), m in zip(ko.block_bounds(F.shape[1], 256), mus))
    W, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    rel = np.linalg.norm(W - Wr) / np.linalg.norm(Wr)
    print(f"row order {order}, {precision}, {sweeps} sweep(s): |shift - mean| max {shift_gap:.3f}, rel-Fro(W) {rel:.3e}")
    assert rel < (W_TOL if precision == "f16x2" else W_TOL_FAST), rel
