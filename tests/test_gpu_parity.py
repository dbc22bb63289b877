"""GPU parity tests (run with -m gpu on an H100): every call goes through the C ABI and is compared with the
fp64 CPU oracle on the same seeded inputs.

Tolerances (stated once, used everywhere below).  The reference computes in fp64 and its suites assert 1e-8 .. 1e-4
(LinearMapperSuite.scala:28-33, BlockWeightedLeastSquaresSuite.scala:115-140, BlockLinearMapperSuite.scala:40-52).
  * parity mode (KS_PRECISION_F16X2, the library default: every MMA operand carried as hi + lo, fp32 accumulation in the
    tensor core, reduced systems assembled and solved in fp64):
      fitted weights rel-Frobenius(W) <= W_TOL = 1e-4 (SURVEY 8d's parity target; on an H100 1.9e-5 / 1.5e-5 at the BASELINE
      shapes of tests/test_gpu_baseline_shapes.py, which gate at 5e-5; what is left is the tensor core's truncating fp32
      accumulation); predictions max-abs <= 1e-4 * max|y|; cosine features <= 2e-5
  * fast modes (one 10-bit-mantissa MMA per product: "f16" on generated features, "tf32"):
      fitted weights rel-Frobenius(W) <= W_TOL_FAST = 1.5e-3 (9.8e-4 on an H100 at the C3 shape); predictions max-abs <= 5e-3
  * Gram kernel alone, operands exactly representable: 5e-5 * sum|a||b| (the tensor core's fp32 accumulation truncates)
"""
import json
import os

import numpy as np
import pytest

import keystone_b200 as ks
from oracle import keystone_oracle as ko

pytestmark = pytest.mark.gpu

W_TOL = 1e-4        # parity mode
W_TOL_FAST = 1.5e-3  # 10-bit operand modes


def round_tf32(x):
    """fp32 -> tf32 with round-to-nearest (ties away), kept in fp32: what cvt.rna.tf32.f32 does on the device."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


def _debug_gram(ctx, A, B):
    import ctypes as C
    from keystone_b200._capi import lib, check
    a, b = ctx.matrix(A.astype(np.float32)), ctx.matrix(B.astype(np.float32))
    m, kc = A.shape[1], B.shape[1]
    G = np.zeros((m, m)); Cm = np.zeros((m, kc))
    check(ctx.handle, lib().ks_debug_gram(ctx.handle, a.handle, b.handle, G.ctypes.data_as(C.c_void_p), m,
                                          Cm.ctypes.data_as(C.c_void_p), kc))
    return G, Cm


@pytest.mark.parametrize("n,m,kc", [(64, 32, 8), (1000, 300, 37), (5000, 640, 257), (40, 12, 3), (9000, 128, 1)])
def test_gram_kernel(ctx, n, m, kc):
    rng = np.random.default_rng(n + m)
    # operands exactly representable in tf32 (the fit always feeds the kernel tf32-rounded slabs): the only error
    # left is the tensor core's fp32 accumulation, which truncates (measured: relative bias ~2.5e-5 on a sum of
    # 9000 positive products, i.e. ~2^-24 per 8-row MMA step); bound: 5e-5 * sum|a||b|
    A = round_tf32(rng.standard_normal((n, m))); B = round_tf32(rng.standard_normal((n, kc)))
    G, Cm = _debug_gram(ctx, A, B)
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    tol_g = 5e-5 * (np.abs(A64).T @ np.abs(A64)).max() + 1e-5
    tol_c = 5e-5 * (np.abs(A64).T @ np.abs(B64)).max() + 1e-5
    assert np.abs(G - A64.T @ A64).max() < tol_g, np.abs(G - A64.T @ A64).max()
    assert np.abs(Cm - A64.T @ B64).max() < tol_c, np.abs(Cm - A64.T @ B64).max()
    # unrounded fp32 operands are truncated by the MMA: bounded by 2^-10 relative per product
    A2 = rng.standard_normal((n, m)).astype(np.float32)
    G2, _ = _debug_gram(ctx, A2, B)
    ref = A2.astype(np.float64).T @ A2.astype(np.float64)
    assert np.abs(G2 - ref).max() < 2.0 ** -9 * np.abs(ref).max()


def test_gram_exact_on_tf32_representable_inputs(ctx):
    """Small integers are exact in tf32 and their sums exact in fp32: the kernel must be bit-exact here,
    which pins the smem/instruction descriptors, the swizzle and the tile masks independently of rounding."""
    rng = np.random.default_rng(7)
    A = rng.integers(-3, 4, (777, 200)).astype(np.float64); B = rng.integers(-3, 4, (777, 70)).astype(np.float64)
    G, Cm = _debug_gram(ctx, A, B)
    assert np.array_equal(G, A.T @ A) and np.array_equal(Cm, A.T @ B)


def test_cosine_random_features(ctx):
    rng = np.random.default_rng(1)
    X = rng.standard_normal((700, 50))
    W, b = ko.cosine_random_features_params(50, 300, 0.3, rng)
    rf = ks.CosineRandomFeatures(ctx, W, b)
    out = rf(ctx.matrix(X)).to_numpy()
    ref = ko.cosine_random_features(X, W, b)
    assert out.shape == ref.shape
    assert np.abs(out - ref).max() < 2e-5, np.abs(out - ref).max()     # reference's own tolerance: 1e-2 (CosineRandomFeaturesSuite.scala:33-35)
    one = rf(X[3])
    assert np.abs(one - ref[3]).max() < 2e-5
    ctx.set_option("precision", 0)                                       # one tf32 MMA per product
    try:
        assert np.abs(rf(ctx.matrix(X)).to_numpy() - ref).max() < 5e-3
    finally:
        ctx.set_option("precision", 2)


def _fit_compare(ctx, F, Y, bs, iters, lam, tol=W_TOL, precision="default"):
    model = ks.BlockLeastSquaresEstimator(bs, iters, lam, precision=precision).fit(ctx.matrix(F), ctx.matrix(Y))
    assert ctx.last_fit_stats()["mma"] == {"default": "tf32x2", "tf32": "tf32x1", "f16": "tf32x1"}[precision]
    # the device stores fp32 inputs: the oracle sees the same values
    F = np.asarray(F, dtype=np.float32).astype(np.float64)
    Y = np.asarray(Y, dtype=np.float32).astype(np.float64)
    xs, b0, mus = ko.block_ls_fit(F, Y, bs, iters, lam)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
    assert [x.shape for x in model.xs] == [x.shape for x in xs]
    assert rel < tol, rel
    assert np.abs(model.b_opt - b0).max() < 1e-6
    # parity mode: column sums of hi + lo; fast modes: of the 10-bit slab (rounding noise ~ 3e-4 rms / sqrt(N))
    mean_tol = (1e-6 if precision == "default" else 5e-5) * max(1.0, np.abs(np.concatenate(mus)).max())
    assert np.abs(np.concatenate(model.feature_means) - np.concatenate(mus)).max() < mean_tol
    return model, xs, b0, mus, rel


def test_blockls_fit_materialized(ctx):
    rng = np.random.default_rng(2)
    n, d, k = 3000, 700, 5
    F = rng.standard_normal((n, d)) + 0.5 * rng.standard_normal(d)   # non-zero column means
    Y = ko.class_label_indicators(rng.integers(0, k, n), k)
    model, xs, b0, mus, rel = _fit_compare(ctx, F, Y, 256, 1, 1.0)
    F32 = F.astype(np.float32).astype(np.float64)
    pred = model(ctx.matrix(F)).to_numpy()
    ref = ko.block_linear_apply(F32, xs, 256, b0, mus)
    assert np.abs(pred - ref).max() < 1e-4, np.abs(pred - ref).max()
    assert (model.apply_argmax(ctx.matrix(F)) == np.argmax(ref, 1)).mean() > 0.9995
    _fit_compare(ctx, F, Y, 256, 1, 1.0, tol=W_TOL_FAST, precision="tf32")


def test_blockls_fit_multi_pass_and_ragged(ctx):
    rng = np.random.default_rng(3)
    n, d, k = 2000, 300, 3
    F = rng.standard_normal((n, d)) * (1 + rng.random(d)) + 1.0
    Y = rng.standard_normal((n, k))
    _fit_compare(ctx, F, Y, 128, 3, 0.5)        # blocks 128,128,44 ; 3 sweeps
    _fit_compare(ctx, F, Y, 300, 1, 0.0)        # nb = 1, lambda = 0 : LinearMapEstimator case
    _fit_compare(ctx, F, Y, 128, 3, 0.5, tol=W_TOL_FAST, precision="tf32")


def test_blockls_fit_reference_fixture(ctx, golden_dir):
    """The reference's aMat/bMat fixture through the GPU BlockLS (b=4, 3 sweeps, lambda 0.1) vs the committed oracle output."""
    A = np.loadtxt(os.path.join(golden_dir, "aMat.csv"), delimiter=",")
    B = np.loadtxt(os.path.join(golden_dir, "bMat.csv"), delimiter=",")
    g = json.load(open(os.path.join(golden_dir, "golden.json")))["block_ls_fixture"]
    model = ks.BlockLeastSquaresEstimator(g["block_size"], g["num_iter"], g["lambda"]).fit(ctx.matrix(A), ctx.matrix(B))
    W = np.concatenate(model.xs, 0)
    assert np.linalg.norm(W - np.array(g["W"])) / np.linalg.norm(g["W"]) < W_TOL
    assert np.abs(model.b_opt - np.array(g["intercept"])).max() < 1e-6


@pytest.mark.parametrize("bs,iters", [(4, 1), (5, 2), (12, 3)])
def test_blockls_pinned_by_weighted_solver_with_zero_mixture_weight(ctx, golden_dir, bs, iters):
    """The identity that pins the BlockLS arithmetic to in-repo reference code (tests/test_oracle_golden.py, same name):
    trainWithL2 with mixtureWeight = 0 (K/nodes/learning/BlockWeightedLeastSquares.scala:216-273) == BlockLS with lambda * N,
    here through the two GPU solvers: ks_blockwls_fit(w = 0) vs ks_blockls_fit(lambda N)."""
    A = np.loadtxt(os.path.join(golden_dir, "aMat.csv"), delimiter=",")
    B = np.loadtxt(os.path.join(golden_dir, "bMat.csv"), delimiter=",")
    n, lam = A.shape[0], 0.1
    mw = ks.BlockWeightedLeastSquaresEstimator(bs, iters, lam, 0.0).fit(ctx.matrix(A), ctx.matrix(B))
    ml = ks.BlockLeastSquaresEstimator(bs, iters, lam * n).fit(ctx.matrix(A), ctx.matrix(B))
    Ww, Wl = np.concatenate(mw.xs, 0), np.concatenate(ml.xs, 0)
    assert np.linalg.norm(Ww - Wl) / np.linalg.norm(Wl) < 2 * W_TOL
    folded = ml.b_opt - sum(mu @ x for mu, x in zip(ml.feature_means, ml.xs))
    assert np.abs(mw.b_opt - folded).max() < 1e-4
    xs, ybar, mus = ko.block_ls_fit(A, B, bs, iters, lam * n)          # and both against the oracle
    assert np.linalg.norm(Wl - np.concatenate(xs, 0)) / np.linalg.norm(np.concatenate(xs, 0)) < W_TOL


def test_blockls_fit_cosine_features_regenerated(ctx):
    """Config-3 shape in miniature: gather(CosineRandomFeatures x3) -> VectorCombiner -> BlockLS, features never stored."""
    rng = np.random.default_rng(4)
    n, d_in, n_out, k = 4000, 44, 256, 10
    X = rng.standard_normal((n, d_in))
    cls = rng.integers(0, k, n)
    params = [ko.cosine_random_features_params(d_in, n_out, 0.17, rng) for _ in range(3)]
    x = ctx.matrix(X.astype(np.float32))
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
    y = ctx.labels_from_classes(cls, k)
    model = ks.BlockLeastSquaresEstimator(n_out, 1, 2.0).fit(feats, y)
    assert ctx.last_fit_stats()["mma"] == "f16x2"
    Xd = X.astype(np.float32).astype(np.float64)
    F = np.concatenate([ko.cosine_random_features(Xd, W, b) for W, b in params], 1)
    Y = ko.class_label_indicators(cls, k)
    xs, b0, mus = ko.block_ls_fit(F, Y, n_out, 1, 2.0)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
    assert rel < W_TOL, rel
    pred = model(feats).to_numpy()
    ref = ko.block_linear_apply(F, xs, n_out, b0, mus)
    assert np.abs(pred - ref).max() < 1e-4
    # computeCost (no centring; BlockLinearMapper.scala:142-187)
    cost = model.compute_cost(feats, y, 2.0)
    assert abs(cost - ko.compute_cost(F, Y, 2.0, xs, n_out, b0)) / cost < 1e-4     # the oracle's cost of the ORACLE's model
    xs_g = [np.array(w) for w in model.xs]
    assert abs(cost - ko.compute_cost(F, Y, 2.0, xs_g, n_out, np.array(model.b_opt))) / cost < 2e-6   # ... and of the GPU's model
    # the tf32 one-MMA mode on the same problem
    m32 = ks.BlockLeastSquaresEstimator(n_out, 1, 2.0, precision="tf32").fit(feats, y)
    assert ctx.last_fit_stats()["mma"] == "tf32x1"
    W32 = np.concatenate(m32.xs, 0)
    assert np.linalg.norm(W32 - Wr) / np.linalg.norm(Wr) < W_TOL_FAST
    # block size different from the feature-map width (blocks straddle maps)
    m2 = ks.BlockLeastSquaresEstimator(200, 1, 2.0).fit(feats, y)
    xs2, _, _ = ko.block_ls_fit(F, Y, 200, 1, 2.0)
    W2, R2 = np.concatenate(m2.xs, 0), np.concatenate(xs2, 0)
    assert np.linalg.norm(W2 - R2) / np.linalg.norm(R2) < W_TOL

# ------------------------------------------------------------------------------------ fp16 operand mode (KS_PRECISION_F16)
@pytest.fixture()
def ctx16(ctx):
    ctx.set_option("precision", 1)
    yield ctx
    ctx.set_option("precision", 2)


@pytest.mark.parametrize("n,m,kc", [(777, 200, 70), (64, 64, 64), (5000, 640, 257), (130, 1030, 5)])
def test_gram_f16_exact_on_small_integers(ctx16, n, m, kc):
    """Small integers are exact in fp16 and their sums exact in fp32: the fp16 wgmma Gram kernel must be bit-exact,
    which pins its MN-major fp16 descriptors (SWIZZLE_128B, LBO = box, SBO = 1024, 2048 B per K = 16 step)."""
    rng = np.random.default_rng(n)
    A = rng.integers(-3, 4, (n, m)).astype(np.float64); B = rng.integers(-3, 4, (n, kc)).astype(np.float64)
    G, Cm = _debug_gram(ctx16, A, B)
    assert np.array_equal(G, A.T @ A), np.abs(G - A.T @ A).max()
    assert np.array_equal(Cm, A.T @ B), np.abs(Cm - A.T @ B).max()


def test_gram_f16_rounding(ctx16):
    rng = np.random.default_rng(11)
    A = rng.standard_normal((3000, 300)).astype(np.float16); B = rng.standard_normal((3000, 40)).astype(np.float16)
    G, Cm = _debug_gram(ctx16, A.astype(np.float64), B.astype(np.float64))
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    assert np.abs(G - A64.T @ A64).max() < 5e-5 * (np.abs(A64).T @ np.abs(A64)).max() + 1e-5
    assert np.abs(Cm - A64.T @ B64).max() < 5e-5 * (np.abs(A64).T @ np.abs(B64)).max() + 1e-5


def _cosine_problem(ctx, seed, n, d_in, n_out, k, n_maps):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d_in))
    cls = rng.integers(0, k, n)
    params = [ko.cosine_random_features_params(d_in, n_out, 0.17, rng) for _ in range(n_maps)]
    x = ctx.matrix(X.astype(np.float32))
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
    Xd = X.astype(np.float32).astype(np.float64)
    F = np.concatenate([ko.cosine_random_features(Xd, W, b) for W, b in params], 1)
    return feats, F, cls


@pytest.mark.parametrize("bs,iters", [(256, 1), (200, 2)])
def test_blockls_fit_f16_matches_oracle(ctx, bs, iters):
    """Same problem and the same tolerance as the tf32 test above, with the fp16 operand path selected per fit."""
    n, k = 4000, 10
    feats, F, cls = _cosine_problem(ctx, 4, n, 44, 256, k, 3)
    y = ctx.labels_from_classes(cls, k)
    Y = ko.class_label_indicators(cls, k)
    model = ks.BlockLeastSquaresEstimator(bs, iters, 2.0, precision="f16").fit(feats, y)
    assert ctx.last_fit_stats()["mma"] == "f16"
    xs, b0, mus = ko.block_ls_fit(F, Y, bs, iters, 2.0)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
    assert rel < W_TOL_FAST, rel
    # the means are those of the generated features (tf32 projection, 10-bit slab): measured 1.2e-4 at N = 4000 in both modes,
    # shrinking like 1/sqrt(N) (4.2e-5 at N = 32768, tools/accuracy_probe.py)
    assert np.abs(np.concatenate(model.feature_means) - np.concatenate(mus)).max() < 5e-4
    pred = model(feats).to_numpy()
    ref = ko.block_linear_apply(F, xs, bs, b0, mus)
    assert np.abs(pred - ref).max() < 5e-3


def test_blockls_fit_f16_label_scale_invariance(ctx):
    """fp16 has a 5-bit exponent: the residual and increment operands carry device-chosen power-of-two scales, so labels of
    magnitude 1e-6 or 1e+5 (far outside fp16's comfortable range) must give the same relative accuracy."""
    n, k = 3000, 4
    feats, F, cls = _cosine_problem(ctx, 9, n, 30, 256, k, 2)
    rng = np.random.default_rng(10)
    Y0 = rng.standard_normal((n, k))
    for scale in (1e-6, 1.0, 1e5):
        Y = Y0 * scale
        model = ks.BlockLeastSquaresEstimator(256, 1, 1.0, precision="f16").fit(feats, ctx.matrix(Y))
        xs, b0, mus = ko.block_ls_fit(F, Y.astype(np.float32).astype(np.float64), 256, 1, 1.0)
        Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
        rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
        assert rel < W_TOL_FAST, (scale, rel)


def test_blockls_fit_f16_input_scale_invariance(ctx):
    """The fp16 projection operands (X and the random-feature weights) carry their own power-of-two scales: inputs in units
    of 1e4 with weights in units of 1e-4 (products unchanged) must fit exactly like the O(1) problem."""
    rng = np.random.default_rng(21)
    n, d_in, n_out, k = 3000, 30, 256, 4
    X = rng.standard_normal((n, d_in))
    cls = rng.integers(0, k, n)
    W, b = ko.cosine_random_features_params(d_in, n_out, 0.2, rng)
    Y = ko.class_label_indicators(cls, k)
    for sx in (1.0, 1e4, 1e-4):
        Xs = (X * sx).astype(np.float32)
        Ws = W / sx
        rf = ks.CosineRandomFeatures(ctx, Ws, b)
        feats = rf(ctx.matrix(Xs))
        model = ks.BlockLeastSquaresEstimator(n_out, 1, 1.0, precision="f16").fit(feats, ctx.labels_from_classes(cls, k))
        assert ctx.last_fit_stats()["mma"] == "f16"
        F = ko.cosine_random_features(Xs.astype(np.float64), Ws.astype(np.float32).astype(np.float64), b)
        xs, _, _ = ko.block_ls_fit(F, Y, n_out, 1, 1.0)
        Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
        rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
        assert rel < W_TOL_FAST, (sx, rel)


@pytest.mark.parametrize("bs,iters", [(256, 1), (200, 2)])
def test_blockls_fit_f16x2_split_operands(ctx, bs, iters):
    """KS_PRECISION_F16X2 (parity mode): same problem as the fp16 test, tolerance 30x tighter (model of the device arithmetic:
    2e-7, tests/test_precision_model.py; the tensor core's truncating fp32 accumulation leaves ~1e-6)."""
    n, k = 4000, 10
    feats, F, cls = _cosine_problem(ctx, 4, n, 44, 256, k, 3)
    y = ctx.labels_from_classes(cls, k)
    Y = ko.class_label_indicators(cls, k)
    model = ks.BlockLeastSquaresEstimator(bs, iters, 2.0, precision="f16x2").fit(feats, y)
    assert ctx.last_fit_stats()["mma"] == "f16x2"
    xs, b0, mus = ko.block_ls_fit(F, Y, bs, iters, 2.0)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
    assert rel < W_TOL, rel
    assert np.abs(np.concatenate(model.feature_means) - np.concatenate(mus)).max() < 5e-6


def test_blockls_parity_mode_scale_invariance(ctx):
    """The split fp16 operands carry device-chosen power-of-two scales (labels, inputs): magnitudes far outside fp16's range
    must not change the relative accuracy of the parity mode."""
    n, k = 3000, 4
    feats, F, cls = _cosine_problem(ctx, 9, n, 30, 256, k, 2)
    rng = np.random.default_rng(10)
    Y0 = rng.standard_normal((n, k))
    for scale in (1e-6, 1.0, 1e5):
        Y = Y0 * scale
        model = ks.BlockLeastSquaresEstimator(256, 1, 1.0).fit(feats, ctx.matrix(Y))
        xs, b0, mus = ko.block_ls_fit(F, Y.astype(np.float32).astype(np.float64), 256, 1, 1.0)
        Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
        rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
        assert rel < W_TOL, (scale, rel)


def test_blockls_f16_falls_back_to_tf32_for_materialized_features(ctx):
    rng = np.random.default_rng(12)
    F = rng.standard_normal((1500, 300)) * 1e4     # far outside fp16's range once squared: must not be computed in fp16
    Y = rng.standard_normal((1500, 3))
    model = ks.BlockLeastSquaresEstimator(128, 1, 1.0, precision="f16").fit(ctx.matrix(F), ctx.matrix(Y))
    assert ctx.last_fit_stats()["mma"] == "tf32x1"
    xs, _, _ = ko.block_ls_fit(F.astype(np.float32).astype(np.float64), Y, 128, 1, 1.0)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    assert np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr) < W_TOL_FAST


def test_linear_map_estimator_known_answer(ctx):
    """T/nodes/learning/LinearMapperSuite.scala:13-36 through the GPU path.  The reference asserts 1e-8 in fp64; the device
    stores its inputs in fp32 (2^-24 relative), so the recoverable accuracy of the planted model is ~1e-6."""
    rng = np.random.default_rng(42)
    A = rng.standard_normal((128, 5)).astype(np.float32).astype(np.float64)   # exactly representable inputs
    x = np.array([5.0, 4.0, 3.0, 2.0, -1.0])[:, None]
    mapper = ks.LinearMapEstimator().fit(ctx.matrix(A), ctx.matrix(A @ x))
    assert ctx.last_fit_stats()["mma"] == "tf32x2"
    assert np.abs(mapper.x - x).max() < 1e-5, np.abs(mapper.x - x).max()
    assert abs(mapper(np.array([2.0, -3.0, 2.0, 3.0, 5.0]))[0] - 5.0) < 1e-4


def test_block_linear_mapper_equals_linear_mapper(ctx):
    """T/nodes/learning/BlockLinearMapperSuite.scala:18-55 on the device, incl. applyAndEvaluate's last callback."""
    rng = np.random.default_rng(5)
    in_dim, out_dim, bs, n = 1000, 100, 200, 50
    mat = rng.standard_normal((in_dim, out_dim)); b = rng.standard_normal(out_dim)
    X = rng.standard_normal((n, in_dim))
    blm = ks.BlockLinearMapper.from_arrays(ctx, [mat[s:e] for s, e in ko.block_bounds(in_dim, bs)], bs, b)
    lm = ks.LinearMapper.from_arrays(ctx, mat, b)
    x = ctx.matrix(X)
    o1, o2 = blm(x).to_numpy(), lm(x).to_numpy()
    ref = X @ mat + b
    scale = np.abs(ref).max()
    # the reference asserts 1e-4 absolute on this shape (BlockLinearMapperSuite.scala:40-52); fp32 inputs: compare against them
    ref = X.astype(np.float32).astype(np.float64) @ mat + b
    assert np.abs(o1 - ref).max() < 1e-5 * scale and np.abs(o2 - ref).max() < 1e-5 * scale
    seen = []
    blm.applyAndEvaluate(x, lambda part: seen.append(part.to_numpy()))
    assert len(seen) == 5 and np.abs(seen[-1] - o1).max() < 1e-5 * scale


def test_error_paths(ctx):
    with pytest.raises(ks.KeystoneError):
        ks.BlockLeastSquaresEstimator(0, 1, 0.0).fit(ctx.matrix(np.ones((4, 4))), ctx.matrix(np.ones((4, 1))))
    with pytest.raises(ks.KeystoneError):
        ks.BlockLeastSquaresEstimator(4, 1, 0.0).fit(ctx.matrix(np.ones((4, 4))), ctx.matrix(np.ones((5, 1))))
    with pytest.raises(ks.KeystoneError):   # singular system, lambda = 0 -> not SPD, reported (no crash / exit)
        ks.BlockLeastSquaresEstimator(4, 1, 0.0).fit(ctx.matrix(np.ones((6, 4))), ctx.matrix(np.ones((6, 1))))


# ---- BlockWeightedLeastSquaresEstimator on the device (T/nodes/learning/BlockWeightedLeastSquaresSuite.scala) ----
def _bwls_compare(ctx, A, B, bs, iters, lam=0.1, w=0.3, tol=W_TOL, precision="default"):
    model = ks.BlockWeightedLeastSquaresEstimator(bs, iters, lam, w, precision=precision).fit(ctx.matrix(A), ctx.matrix(B))
    assert ctx.last_fit_stats()["mma"] == ("tf32x2" if precision == "default" else "tf32x1")
    xs, fb = ko.bwls_fit(A, B, bs, iters, lam, w)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    assert [x.shape for x in model.xs] == [x.shape for x in xs]
    assert model.feature_means is None                       # no feature scalers (BlockWeightedLeastSquares.scala:320)
    err, ref = np.linalg.norm(Wg - Wr), np.linalg.norm(Wr)
    assert err <= tol * ref + 1e-6, (err, ref)      # the single-class fixture has W == 0 exactly
    assert np.abs(model.b_opt - fb).max() < tol * max(1.0, np.abs(fb).max())
    return model, Wg, Wr, fb


def test_bwls_reference_fixture(ctx, golden_dir):
    """:142-166 (b=4, 10 iters, gradient of the weighted objective ~ 0) and :188-223 (ragged b=5) on aMat/bMat."""
    A = np.loadtxt(os.path.join(golden_dir, "aMat.csv"), delimiter=",")
    B = np.loadtxt(os.path.join(golden_dir, "bMat.csv"), delimiter=",")
    model, Wg, Wr, fb = _bwls_compare(ctx, A, B, 4, 10)
    g = ko.compute_gradient(A, B, 0.1, 0.3, Wg, model.b_opt)
    g_ref = ko.compute_gradient(A, B, 0.1, 0.3, Wr, fb)
    # the reference bound is 1e-2 and the fp64 oracle sits at 8.1e-3
    assert np.linalg.norm(g) < np.linalg.norm(g_ref) + 1e-4
    _bwls_compare(ctx, A, B, 4, 10, tol=5e-3, precision="tf32")
    model5, W5, _, _ = _bwls_compare(ctx, A, B, 5, 10)
    assert np.linalg.norm(ko.compute_gradient(A, B, 0.1, 0.3, W5, model5.b_opt)) < 1e-1
    # predictions through BlockLinearMapper.apply (no scalers, intercept = finalB)
    pred = model(ctx.matrix(A)).to_numpy()
    assert np.abs(pred - (A @ Wr + fb)).max() < 1e-4


def test_bwls_group_by_classes_and_degenerate_cases(ctx, golden_dir):
    """:225-253 (rows not grouped by class -> reshuffled on the device), :72-113 (a class with no rows), :168-186 (one class)."""
    A = np.loadtxt(os.path.join(golden_dir, "aMatShuffled.csv"), delimiter=",")
    B = np.loadtxt(os.path.join(golden_dir, "bMatShuffled.csv"), delimiter=",")
    _bwls_compare(ctx, A, B, 4, 10)
    stats = ctx.last_fit_stats()
    assert stats["solver"] == "blockwls" and stats["reshuffled"] == 1
    A0 = np.loadtxt(os.path.join(golden_dir, "aMat.csv"), delimiter=",")
    B0 = np.loadtxt(os.path.join(golden_dir, "bMat.csv"), delimiter=",")
    keep = np.r_[0:5, 10:15]                                   # class 1 has no rows
    m, Wg, Wr, fb = _bwls_compare(ctx, A0[keep], B0[keep], 4, 10)
    assert np.all(Wg[:, 1] == 0.0)
    A1 = np.loadtxt(os.path.join(golden_dir, "aMat-1class.csv"), delimiter=",")
    B1 = np.loadtxt(os.path.join(golden_dir, "bMat-1class.csv"), delimiter=",", ndmin=2)
    _bwls_compare(ctx, A1, B1, 4, 10)


def test_bwls_larger_problem_cosine_features(ctx):
    """Class-imbalanced synthetic problem, features generated on the fly, 2 passes."""
    rng = np.random.default_rng(9)
    n, d_in, n_out, k = 3000, 30, 128, 5
    X = rng.standard_normal((n, d_in))
    cls = np.sort(rng.choice(k, n, p=[0.4, 0.25, 0.2, 0.1, 0.05]))
    params = [ko.cosine_random_features_params(d_in, n_out, 0.25, rng) for _ in range(2)]
    x = ctx.matrix(X.astype(np.float32)); y = ctx.labels_from_classes(cls, k)
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
    model = ks.BlockWeightedLeastSquaresEstimator(n_out, 2, 0.01, 0.25).fit(feats, y)
    Xd = X.astype(np.float32).astype(np.float64)
    F = np.concatenate([ko.cosine_random_features(Xd, W, b) for W, b in params], 1)
    xs, fb = ko.bwls_fit(F, ko.class_label_indicators(cls, k), n_out, 2, 0.01, 0.25)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    assert np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr) < 5e-4    # lambda = 0.01 on n_c as small as 150: conditioning ~1e3
    pred = model(feats).to_numpy()
    ref = F @ Wr + fb
    assert np.abs(pred - ref).max() < 5e-4


@pytest.mark.parametrize("n,k", [(4096, 1000), (4096, 125), (4096, 250), (4096, 500), (300, 37), (128, 8), (5, 3), (1000, 1), (777, 130),
                                 (1000, 1057), (4096, 2000)])   # k > 8 * 132: chol_solve_kernel<16>
def test_chol_solve_kernel(ctx, n, k):
    """The library's DMMA multi-RHS Cholesky solve (one launch; clusters of 2 / 4 / 8 CTAs per column group when there are few
    right-hand sides, as in the column-sharded multi-GPU solve) vs numpy, and vs cuSOLVER."""
    import ctypes as C
    from keystone_b200._capi import lib, check
    rng = np.random.default_rng(n + k)
    A = rng.standard_normal((n + 50, n))
    H = np.asfortranarray(A.T @ A + 0.5 * np.eye(n))
    B = np.asfortranarray(rng.standard_normal((n, k)))
    ref = np.linalg.solve(H, B)
    out = {}
    for use_cusolver in (0, 1):
        X = np.empty((n, k), order="F"); ms = C.c_double(0)
        check(ctx.handle, lib().ks_debug_chol_solve(ctx.handle, H.ctypes.data_as(C.c_void_p), n, B.ctypes.data_as(C.c_void_p), k,
                                                   use_cusolver, X.ctypes.data_as(C.c_void_p), C.byref(ms)))
        out[use_cusolver] = (X, ms.value)
        assert np.abs(X - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()) * np.linalg.cond(H)
    print(f"chol_solve n={n} k={k}: kernel {out[0][1]:.3f} ms, cusolver potrs {out[1][1]:.3f} ms")


def test_device_confusion_matrix_matches_oracle(ctx):
    """ks_model_confusion_matrix: apply -> MaxClassifier -> counts on the device vs the oracle's confusion matrix of the same
    predictions (integer counts: exact)."""
    rng = np.random.default_rng(31)
    n, d, k = 5000, 60, 7
    F = rng.standard_normal((n, d))
    cls = rng.integers(0, k, n)
    Y = ko.class_label_indicators(cls, k)
    model = ks.BlockLeastSquaresEstimator(32, 1, 1.0).fit(ctx.matrix(F), ctx.matrix(Y))
    pred = model.apply_argmax(ctx.matrix(F))
    metrics = ks.MulticlassClassifierEvaluator(k).evaluate_model(model, ctx.matrix(F), ctx.matrix(Y))
    ref = ko.confusion_matrix(pred, cls, k)
    assert np.array_equal(metrics.confusionMatrix, ref)
    assert metrics.confusionMatrix.sum() == n
    assert abs(metrics.totalAccuracy - (pred == cls).mean()) < 1e-12



# ---- MNIST random-FFT featurizer on the device (SURVEY 8f next-3) ------------------------------------------------------
def test_padded_fft_known_answers_on_device(ctx):
    """T/nodes/stats/PaddedFFTSuite.scala:13-36 through the cosine-matrix GEMM."""
    ones = np.zeros(100); ones[0] = 1.0
    twos = np.zeros(100); twos[2] = 1.0
    out = ks.PaddedFFT(ctx)(ctx.matrix(np.stack([twos, ones]))).to_numpy()
    assert out.shape == (2, 64)
    assert abs(out[0, 0] - 1.0) < 1e-6 and abs(out[0, 16]) < 1e-6 and abs(out[0, 32] + 1.0) < 1e-6 and abs(out[0, 48]) < 1e-6
    assert np.abs(out[1] - 1.0).max() < 1e-6


def test_random_sign_and_rectifier_nodes_on_device(ctx):
    """RandomSignNodeSuite.scala:11-18, LinearRectifierSuite.scala:13-27 (elementwise nodes on a batch)."""
    out = ks.RandomSignNode(np.array([1.0, -1.0, 1.0]), ctx)(ctx.matrix(np.array([[1.0, 2.0, 3.0]]))).to_numpy()
    assert np.array_equal(out, np.array([[1.0, -2.0, 3.0]]))
    x = np.random.default_rng(0).standard_normal((128, 16))
    y = ks.LinearRectifier(ctx=ctx)(ctx.matrix(x)).to_numpy()
    assert (x < 0).any() and (y >= 0).all()
    assert np.array_equal(y, np.maximum(0.0, x.astype(np.float32).astype(np.float64)))
    node = ks.RandomSignNode.create(1000, np.random.default_rng(1))
    assert set(np.unique(node.signs)) <= {-1.0, 1.0}


def test_mnist_random_fft_pipeline_matches_oracle(ctx):
    """MnistRandomFFT.scala:40-47 in miniature: gather(RandomSignNode -> PaddedFFT -> LinearRectifier) x 4 -> VectorCombiner
    -> BlockLeastSquaresEstimator(blockSize, 1, lambda) -> MaxClassifier; features (fused FFT GEMM + rectifier epilogue),
    fitted model and predictions against the oracle."""
    rng = np.random.default_rng(3)
    n, d_in, num_ffts, k, bs, lam = 3000, 784, 4, 10, 1024, 10.0
    X = rng.random((n, d_in)).astype(np.float32)                    # pixel-scale inputs
    cls = rng.integers(0, k, n)
    signs = [2.0 * rng.integers(0, 2, d_in) - 1.0 for _ in range(num_ffts)]
    x = ctx.matrix(X)
    branches = [ks.RandomSignNode(s, ctx).andThen(ks.PaddedFFT(ctx)).andThen(ks.LinearRectifier(0.0, ctx=ctx)) for s in signs]
    feats = ks.Pipeline.gather(branches).andThen(ks.VectorCombiner())(x)
    assert feats.shape == (n, num_ffts * 512)
    F = ko.mnist_random_fft_features(X.astype(np.float64), signs)
    Fg = feats.to_numpy()
    assert np.abs(Fg - F).max() < 1e-4 * np.abs(F).max()
    y = ctx.labels_from_classes(cls, k)
    model = ks.BlockLeastSquaresEstimator(bs, 1, lam).fit(feats, y)
    assert ctx.last_fit_stats()["mma"] == "tf32x2"                   # rectified features have the scale of their input: tf32 pairs
    xs, b0, mus = ko.block_ls_fit(F, ko.class_label_indicators(cls, k), bs, 1, lam)
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    assert np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr) < W_TOL
    ref = ko.block_linear_apply(F, xs, bs, b0, mus)
    pred = model.apply_argmax(feats)
    assert (pred == np.argmax(ref, 1)).mean() > 0.999
    mfast = ks.BlockLeastSquaresEstimator(bs, 1, lam, precision="f16").fit(feats, y)
    assert ctx.last_fit_stats()["mma"] == "tf32x1"
    # one tf32 MMA per product on this ill-conditioned problem (all-positive pixel sums: every FFT feature correlates with the DC
    # bin; lambda = 10 against Gram entries of ~1e6): the 10-bit operand noise is amplified, only sanity is asserted
    rel_fast = np.linalg.norm(np.concatenate(mfast.xs, 0) - Wr) / np.linalg.norm(Wr)
    print(f"MNIST-FFT fast mode rel-Fro(W) = {rel_fast:.3e}")
    assert rel_fast < 0.2


def test_model_save_load_round_trip(ctx, tmp_path):
    """Fitted model -> flat file -> model (replaces the Java-serialised FittedPipeline, K/workflow/FittedPipeline.scala:18-22):
    bit-identical arrays and identical predictions; a BWLS model (no feature scalers) survives too."""
    rng = np.random.default_rng(8)
    F = rng.standard_normal((500, 70)); Y = rng.standard_normal((500, 3))
    f = ctx.matrix(F)
    m = ks.BlockLeastSquaresEstimator(32, 1, 1.0).fit(f, ctx.matrix(Y))
    p = str(tmp_path / "model.ksb")
    m.save(p)
    m2 = ks.BlockLinearMapper.load(ctx, p)
    assert m2.num_blocks == 3 and m2.k == 3 and m2.block_size == 32
    assert all(np.array_equal(a, b) for a, b in zip(m.xs, m2.xs))
    assert all(np.array_equal(a, b) for a, b in zip(m.feature_means, m2.feature_means))
    assert np.array_equal(m.b_opt, m2.b_opt)
    assert np.array_equal(m(f).to_numpy(), m2(f).to_numpy())
    cls = rng.integers(0, 3, 500)
    mw = ks.BlockWeightedLeastSquaresEstimator(32, 1, 0.1, 0.3).fit(f, ctx.labels_from_classes(cls, 3))
    mw.save(p)
    mw2 = ks.BlockLinearMapper.load(ctx, p)
    assert mw2.feature_means is None and np.array_equal(mw.b_opt, mw2.b_opt)
    assert all(np.array_equal(a, b) for a, b in zip(mw.xs, mw2.xs))
    with pytest.raises(ks.KeystoneError):
        (tmp_path / "junk").write_bytes(b"not a model")
        ks.BlockLinearMapper.load(ctx, str(tmp_path / "junk"))


# ---- CIFAR random-patch featurizer on the device (SURVEY 8f next-1) ----------------------------------------------------
def test_convolver_matches_reference_golden_image_on_device(ctx, golden_dir):
    """T/nodes/images/ConvolverSuite.scala:100-137 through the device path: crops of the reference's test image (the image itself
    exceeds the one-image-per-CTA shared-memory window) convolved with the suite's two 3 x 3 x 3 filters, flipFilters = true, no
    normalisation; channel 0 must equal the matching crop of convolved.gantrycrane.csv EXACTLY (integer arithmetic survives the
    fp16 operands: pixels <= 255, filter taps <= 26, fp32 accumulation)."""
    z = np.load(os.path.join(golden_dir, "conv_gantrycrane.npz"))
    img, expected = ko.image_from_bgr_bytes(z["rgb"]), z["expected"].astype(np.float64)
    kimg, kimg2 = np.zeros((3, 3, 3)), np.zeros((3, 3, 3))
    i = 0
    for x in range(3):
        for y in range(3):
            for c in range(3):
                kimg[x, y, 2 - c] = float(i)
                i += 1
    kimg2[0, 0, 0] = 2.0
    kimg2[2, 0, 1] = 1.0
    filt = np.zeros((4, 27))                                              # two zero filters: the output row stride must be 16 B aligned
    filt[:2] = ko.pack_filters([ko.flip_image(kimg), ko.flip_image(kimg2)])
    S = 34                                                                 # 34 x 34 crops -> 32 x 32 outputs
    offs = [(0, 0), (100, 200), (230, 366), (57, 123)]
    crops = np.stack([img[a:a + S, b:b + S, :] for a, b in offs])
    conv = ks.Convolver(ctx, filt, S, S, 3, None, normalize_patches=False)
    out = conv(ctx.matrix(ks.images_to_matrix(crops))).to_numpy()
    assert out.shape == (4, 32 * 32 * 4)
    for n, (a, b) in enumerate(offs):
        got = np.transpose(out[n].reshape(32, 32, 4), (1, 0, 2))          # vectorised order c + x*C + y*C*xDim -> [x, y, c]
        assert np.array_equal(got[:, :, 0], expected[a:a + 32, b:b + 32]), (n, np.abs(got[:, :, 0] - expected[a:a + 32, b:b + 32]).max())
        assert np.array_equal(got[:, :, 1], ko.convolve(crops[n], filt, 3, normalize=False)[:, :, 1])


def test_cifar_random_patch_featurizer_matches_oracle(ctx):
    """RandomPatchCifar.scala:59-63 in miniature: Convolver(whitened filters, whitener means, normalizePatches) andThen
    SymmetricRectifier(alpha = 0.25) andThen Pooler(13, 14, identity, sum) andThen ImageVectorizer on CIFAR-shaped images (32 x 32 x 3,
    6 x 6 patches -> 27 x 27 responses -> 2 x 2 overlapping pools), fused on the device, vs the oracle; then the same features through
    BlockLeastSquaresEstimator with the pipeline's ragged last block."""
    rng = np.random.default_rng(5)
    n, nf, k = 96, 160, 10
    imgs = rng.integers(0, 256, (n, 32, 32, 3)).astype(np.float64)         # [n][x][y][c]
    filters = rng.standard_normal((nf, 108)) / 10.0
    wmeans = rng.standard_normal(108) * 0.05
    conv = ks.Convolver(ctx, filters, 32, 32, 3, wmeans, normalize_patches=True, var_constant=10.0)
    chain = conv.andThen(ks.SymmetricRectifier(alpha=0.25)).andThen(ks.Pooler(13, 14)).andThen(ks.ImageVectorizer())
    feats = chain(ctx.matrix(ks.images_to_matrix(imgs)))
    assert feats.shape == (n, 2 * 2 * 2 * nf)
    ref = np.stack([ko.random_patch_cifar_features(im, filters, wmeans, 6, 0.25, 13, 14) for im in imgs])
    got = feats.to_numpy()
    assert np.abs(got - ref).max() < 1e-4 * np.abs(ref).max(), np.abs(got - ref).max() / np.abs(ref).max()
    ctx.set_option("precision", 1)                                           # one fp16 MMA per product
    try:
        fast = chain(ctx.matrix(ks.images_to_matrix(imgs))).to_numpy()
    finally:
        ctx.set_option("precision", 2)
    assert np.abs(fast - ref).max() < 5e-3 * np.abs(ref).max()
    cls = rng.integers(0, k, n)
    model = ks.BlockLeastSquaresEstimator(512, 1, 3000.0).fit(feats, ctx.labels_from_classes(cls, k))
    xs, b0, mus = ko.block_ls_fit(got, ko.class_label_indicators(cls, k), 512, 1, 3000.0)
    assert [w.shape[0] for w in model.xs] == [512, 512, 256]
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    assert np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr) < W_TOL


def test_cifar_loader_layout_feeds_the_convolver(ctx):
    """CifarLoader's channel planes (K/loaders/CifarLoader.scala:20-28) -> Convolver input rows: a one-hot image must light up the
    patch column the reference's makePatches assigns it."""
    planes = np.zeros((1, 3, 32, 32), dtype=np.uint8)
    planes[0, 2, 5, 7] = 200                                                 # channel 2, x = 5, y = 7
    row = ks.cifar_bytes_to_matrix(planes)
    img = np.transpose(planes[0].astype(np.float64), (1, 2, 0))              # [x, y, c]
    assert np.array_equal(row[0], ko.image_vectorizer(img).astype(np.float32))
    filt = np.eye(108)[:32]                                                  # filter f responds to patch column f
    out = ks.Convolver(ctx, filt, 32, 32, 3, None, normalize_patches=False)(ctx.matrix(row)).to_numpy()
    ref = ko.convolve(img, filt, 6, normalize=False)
    assert np.array_equal(np.transpose(out[0].reshape(27, 27, 32), (1, 0, 2)), ref)


def test_least_squares_estimator_runs_the_selected_gpu_solver(ctx):
    """K/nodes/learning/LeastSquaresEstimator.scala:63-87: the cost model picks a solver from (n, d, k, sparsity, machines) and the
    fit runs it -- here the exact solver (LinearMapEstimator) for a small dense problem, checked against the oracle's closed form."""
    rng = np.random.default_rng(17)
    F = rng.standard_normal((2000, 60)); Y = rng.standard_normal((2000, 4))
    est = ks.LeastSquaresEstimator(lam=0.5, num_machines=1, ctx=ctx)
    model = est.fit(ctx.matrix(F), ctx.matrix(Y))
    assert est.selected == "exact" and est.used == "exact"
    x, ymu, mu = ko.linear_map_fit(F.astype(np.float32).astype(np.float64), Y.astype(np.float32).astype(np.float64), 0.5)
    assert np.linalg.norm(model.xs[0] - x) / np.linalg.norm(x) < W_TOL
    assert np.abs(model.b_opt - ymu).max() < 1e-6
