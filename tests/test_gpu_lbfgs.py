"""Dense L-BFGS least squares (DenseLBFGSwithL2) on the H100 through the C ABI / node API, against the fp64 oracle
(tests/lbfgs_oracle.py) on the same fp32-rounded inputs.

Gates: rel-Frobenius(W) <= W_TOL = 1e-4 and loss history relative <= 1e-6 in the parity mode (every MMA operand a hi + lo pair),
1.5e-3 for both in the fast mode (one 10-bit-mantissa MMA per product), the project's tolerances.  Every fitted problem has
cond(A_c^T A_c / N + lambda I) <= 100 (lambda is chosen from the spectrum where the data alone does not guarantee it)."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import lbfgs_oracle as lo  # noqa: E402

W_TOL, W_TOL_FAST = 1e-4, 1.5e-3


@pytest.fixture(scope="module")
def ctx():
    import keystone_b200 as ks
    c = ks.Context(0)
    yield c
    c.close()


def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


def _lam_for_cond(A, fit_intercept, cond=99.0):
    """reg_param with cond(A_c^T A_c / N + lambda I) <= cond + 1."""
    Ac = A - A.mean(0) if fit_intercept else A
    ev = np.linalg.eigvalsh(Ac.T @ Ac / A.shape[0])
    return max(0.0, (ev[-1] - cond * ev[0]) / (cond - 1.0)) + 1e-12


# ---------------------------------------------------------------------------------------------------------- 1. known answers
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_suite_known_answers(ctx, fit_intercept):
    """T/nodes/learning/LBFGSSuite.scala:13-60 at the default parameters: predictions, W, intercept and means within 1e-5."""
    import keystone_b200 as ks
    A, B, x, data_mean, extra_bias = lo.suite_data(fit_intercept)
    est = ks.DenseLBFGSwithL2(ks.LeastSquaresDenseGradient(), fit_intercept=fit_intercept, ctx=ctx)
    mapper = est.fit(A.astype(np.float32), B.astype(np.float32))
    assert isinstance(mapper, ks.LinearMapper)
    assert np.abs(mapper.apply(A.astype(np.float32)).to_numpy() - B).max() < 1e-5
    assert np.abs(mapper.x - x.T).max() < 1e-5
    if fit_intercept:
        assert np.abs(mapper.b_opt - extra_bias).max() < 1e-5
        assert np.abs(mapper.feature_means[0] - data_mean).max() < 1e-5
    else:
        assert mapper.b_opt is None and mapper.feature_means is None
    assert est.iterations >= 1 and len(est.loss_history) == est.iterations + 1
    assert est.stop_reason in ("gradient_converged", "function_values_converged", "max_iterations")


# ---------------------------------------------------------------------------------------------------------- 2. iterate parity
@pytest.mark.parametrize("precision", ["f16x2", "f16"])
@pytest.mark.parametrize("n,d,k,fit_intercept", [(5000, 4197, 1, True), (4999, 4197, 7, False), (1001, 300, 7, True)])
def test_materialised_iterates_match_oracle(ctx, precision, n, d, k, fit_intercept):
    """8 steps with convergence_tol = 0 on materialised features (D not a multiple of 128 or 4096: a ragged second block)."""
    import keystone_b200 as ks
    rng = np.random.default_rng(n + d + k)
    # offsets only where the fit centres them: without intercept, features or labels with a large mean make the products' fp32
    # accumulation (in the tensor core and in the residual) lose digits to cancellation that no operand precision recovers
    off = 1.0 if fit_intercept else 0.0
    A = _f32(rng.standard_normal((n, d)) * np.linspace(0.5, 1.5, d) + 0.7 * off)
    Y = _f32(A @ rng.standard_normal((d, k)) / np.sqrt(d) + 0.5 * rng.standard_normal((n, k)) + 2.0 * off)
    lam = _lam_for_cond(A, fit_intercept)
    est = ks.DenseLBFGSwithL2(fit_intercept=fit_intercept, num_corrections=5, convergence_tol=0.0, num_iterations=8, reg_param=lam,
                              ctx=ctx, precision=precision)
    mapper = est.fit(A.astype(np.float32), Y.astype(np.float32))
    W, b, mu, info = lo.fit(A, Y, fit_intercept, 5, 0.0, 8, lam)
    assert est.iterations == 8 and est.stop_reason == "max_iterations"
    assert ctx.last_fit_stats()["mma"] == ("tf32x2" if precision == "f16x2" else "tf32x1")
    assert ctx.last_fit_stats()["loss_history"] == est.loss_history
    tol_w, tol_f = (W_TOL, 1e-6) if precision == "f16x2" else (W_TOL_FAST, W_TOL_FAST)
    Wg = np.concatenate(mapper.xs, 0)
    assert mapper.x.shape == (d, k) and np.array_equal(mapper.x, Wg)   # the LinearMapper's one W, whatever the feature blocks
    assert _rel(Wg, W) <= tol_w, _rel(Wg, W)
    lh = np.array(est.loss_history)
    assert np.abs(lh - info["loss_history"]).max() / np.abs(info["loss_history"]).max() <= tol_f
    if fit_intercept:
        assert len(mapper.feature_means) == 1 and mapper.feature_means[0].shape == (d,)
        assert np.abs(mapper.feature_means[0] - mu).max() < 1e-6
        assert np.abs(mapper.b_opt - b).max() < 1e-6


def _cosine(ctx, seed, n, d_in, outs):
    import keystone_b200 as ks
    from oracle import keystone_oracle as ko
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d_in)).astype(np.float32)
    params = [ko.cosine_random_features_params(d_in, m, 0.6 / np.sqrt(d_in), rng) for m in outs]
    x = ctx.matrix(X)
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
    F = np.concatenate([ko.cosine_random_features(X.astype(np.float64), W, b) for W, b in params], 1)
    return feats, F, rng


@pytest.mark.parametrize("precision", ["f16x2", "f16"])
def test_generated_iterates_match_oracle(ctx, precision):
    """x_in + 2 cosine maps (4300 features: a ragged second block), regenerated for every product."""
    import keystone_b200 as ks
    n, k = 6001, 7
    feats, F, rng = _cosine(ctx, 3, n, 40, [1900, 2400])
    Y = _f32(F @ rng.standard_normal((F.shape[1], k)) / 30 + 0.3 * rng.standard_normal((n, k)))
    lam = _lam_for_cond(F, True)
    est = ks.DenseLBFGSwithL2(num_corrections=4, convergence_tol=0.0, num_iterations=8, reg_param=lam, ctx=ctx, precision=precision)
    mapper = est.fit(feats, ctx.matrix(Y.astype(np.float32)))
    assert ctx.last_fit_stats()["mma"] == precision
    W, b, mu, info = lo.fit(F, Y, True, 4, 0.0, 8, lam)
    tol_w, tol_f = (W_TOL, 1e-6) if precision == "f16x2" else (W_TOL_FAST, W_TOL_FAST)
    assert _rel(np.concatenate(mapper.xs, 0), W) <= tol_w
    lh = np.array(est.loss_history)
    assert np.abs(lh - info["loss_history"]).max() / np.abs(info["loss_history"]).max() <= tol_f
    # the exact means are the sample estimate plus the column sums of the stored slab: fp16 pairs here, plain fp16 in the fast mode
    assert np.abs(np.concatenate(mapper.feature_means) - mu).max() < (5e-6 if precision == "f16x2" else 2e-4)


# ---------------------------------------------------------------------------------------------------------- 3. converged fit
def test_converged_fit_equals_linear_map_estimator(ctx):
    """min f with reg_param lambda is LinearMapEstimator(N lambda) (both on the device)."""
    import keystone_b200 as ks
    rng = np.random.default_rng(11)
    n, d, k = 4000, 257, 3
    A = _f32(rng.standard_normal((n, d)) + 1.0)
    Y = _f32(A @ rng.standard_normal((d, k)) / 16 + 0.2 * rng.standard_normal((n, k)))
    lam = _lam_for_cond(A, True, 50.0)
    est = ks.DenseLBFGSwithL2(convergence_tol=1e-12, num_iterations=300, reg_param=lam, ctx=ctx)
    W = est.fit(A.astype(np.float32), Y.astype(np.float32)).x
    Wd = ks.LinearMapEstimator(n * lam, ctx=ctx).fit(ctx.matrix(A.astype(np.float32)), ctx.matrix(Y.astype(np.float32))).x
    assert _rel(W, Wd) <= 1e-4, (_rel(W, Wd), est.stop_reason, est.iterations)
    assert _rel(W, lo.ridge(A, Y, n * lam)) <= 1e-4


def test_stats_of_a_long_fit(ctx):
    """The loss history of a 400-step fit makes the stats JSON far longer than 4 KB; Context.last_fit_stats sizes its buffer."""
    import keystone_b200 as ks
    rng = np.random.default_rng(12)
    A = (rng.standard_normal((600, 80)) * np.logspace(-2, 0, 80)).astype(np.float32)   # slow convergence with one pair
    Y = rng.standard_normal((600, 2)).astype(np.float32)
    est = ks.DenseLBFGSwithL2(num_corrections=1, convergence_tol=0.0, num_iterations=400, reg_param=1e-6, ctx=ctx)
    est.fit(A, Y)
    st = ctx.last_fit_stats()
    assert st["solver"] == "lbfgs" and st["iterations"] == est.iterations
    assert st["loss_history"] == est.loss_history
    from keystone_b200._capi import lib
    n = C.c_int64(0)
    assert lib().ks_last_fit_stats_json_size(ctx.handle, C.byref(n)) == 0
    assert n.value > 4096 or est.iterations < 150, (n.value, est.iterations, est.stop_reason)


# ---------------------------------------------------------------------------------------------------------- 4. the model
def test_model_apply_save_load_cost(ctx, tmp_path):
    import keystone_b200 as ks
    rng = np.random.default_rng(4)
    n, d, k = 2000, 150, 5
    A = _f32(rng.standard_normal((n, d)) + 0.5)
    cls = rng.integers(0, k, n)
    Y = -np.ones((n, k)); Y[np.arange(n), cls] = 1.0
    est = ks.DenseLBFGSwithL2(num_iterations=30, reg_param=1e-3, ctx=ctx)
    m = est.fit(A.astype(np.float32), Y.astype(np.float32))
    W, b, mu = m.x, m.b_opt, m.feature_means[0]
    pred = m.apply(A.astype(np.float32)).to_numpy()
    ref = lo.apply(W, b, mu, A)
    assert np.abs(pred - ref).max() <= 1e-4 * np.abs(ref).max()
    assert np.mean(m.apply_argmax(A.astype(np.float32)) == np.argmax(ref, 1)) > 0.999
    path = str(tmp_path / "lbfgs.ksm")
    m.save(path)
    m2 = ks.LinearMapper.load(ctx, path)
    assert np.array_equal(m2.x, W) and np.array_equal(m2.b_opt, b) and np.array_equal(m2.feature_means[0], mu)
    assert np.abs(m2.apply(A.astype(np.float32)).to_numpy() - pred).max() <= 1e-6 * np.abs(pred).max()
    # computeCost applies no feature scalers (BlockLinearMapper.scala:142-187)
    cost = m.compute_cost(A.astype(np.float32), Y.astype(np.float32), 0.1)
    ref_cost = ((A @ W + b - Y) ** 2).sum() / (2 * n) + 0.05 * (W ** 2).sum()
    assert abs(cost - ref_cost) <= 1e-4 * ref_cost


# ---------------------------------------------------------------------------------------------------------- 5. rejections
def test_rejections(ctx):
    import keystone_b200 as ks
    from keystone_b200._capi import lib
    f = ctx.matrix(np.ones((10, 3), dtype=np.float32))
    y = ctx.matrix(np.ones((10, 2), dtype=np.float32))
    y_bad = ctx.matrix(np.ones((9, 2), dtype=np.float32))
    h = C.c_int64(0)

    def call(labels=y.handle, m=10, tol=1e-4, iters=100, lam=0.0, prec=-1):
        return lib().ks_lbfgs_fit(ctx.handle, f.handle, 0, None, 0, labels, 1, m, tol, iters, lam, prec, C.byref(h))

    assert call() == 0
    ks.LinearMapper(ctx, h.value)   # owns and frees the handle
    for kw in [dict(m=0), dict(iters=0), dict(lam=-1.0), dict(lam=float("nan")), dict(lam=float("inf")), dict(tol=-1.0),
               dict(tol=float("nan")), dict(labels=y_bad.handle), dict(prec=7)]:
        assert call(**kw) == -1, kw
    with pytest.raises(ks.KeystoneError):
        ks.DenseLBFGSwithL2(ctx=ctx).fit(f, y_bad)


# ---------------------------------------------------------------------------------------------------------- 6. two ranks
def _worker(rank, world, id_holder, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import keystone_b200 as ks
    rng = np.random.default_rng(8)
    n, d, k = 3001, 4500, 3
    A = rng.standard_normal((n, d)).astype(np.float32) + 0.3
    Y = (A[:, :40] @ rng.standard_normal((40, k)) + rng.standard_normal((n, k))).astype(np.float32)
    rows = np.r_[0:1000] if rank == 0 else np.r_[1000:n]   # uneven shards
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    est = ks.DenseLBFGSwithL2(num_iterations=8, convergence_tol=0.0, reg_param=0.5, ctx=ctx)
    m = est.fit(A[rows], Y[rows])
    ret[f"W{rank}"] = np.concatenate(m.xs, 0)
    ret[f"b{rank}"] = m.b_opt
    ret[f"mu{rank}"] = np.concatenate(m.feature_means)
    ret[f"loss{rank}"] = est.loss_history
    ctx.close()
    if rank == 0:
        c1 = ks.Context(device=0)
        e1 = ks.DenseLBFGSwithL2(num_iterations=8, convergence_tol=0.0, reg_param=0.5, ctx=c1)
        ret["W1rank"] = np.concatenate(e1.fit(A, Y).xs, 0)
        ret["loss1rank"] = e1.loss_history
        c1.close()


def test_two_rank_fit_equals_one_rank():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import keystone_b200 as ks
    mgr = mp.Manager()
    id_holder = mgr.dict(); ret = mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    assert np.array_equal(ret["W0"], ret["W1"]) and np.array_equal(ret["b0"], ret["b1"]) and np.array_equal(ret["mu0"], ret["mu1"])
    assert ret["loss0"] == ret["loss1"]
    assert _rel(ret["W0"], ret["W1rank"]) <= 1e-4
    assert np.allclose(ret["loss0"], ret["loss1rank"], rtol=1e-6, atol=0)
