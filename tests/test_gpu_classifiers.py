"""Logistic regression and multinomial naive Bayes (LogisticRegressionEstimator, NaiveBayesEstimator) on the H100, against the fp64
oracle of tests/classifier_oracle.py (DESIGN.md section 22).

Both fits are fp64 after the features (dense inputs are fp32 matrices; the oracle gets the same fp32-rounded values), so only
summation order differs: rel-Frobenius(W) <= 1e-9, loss history within 1e-11 of f(W_0) = log k, and the same line-search
evaluation counts and stop reason.  Every iterate case stops by max_iterations well before convergence to rounding."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import classifier_oracle as co  # noqa: E402
from test_oracle_classifiers import (NB_PI, NB_THETA, MULTI_WEIGHTS_R, logistic_input, multinomial_input,  # noqa: E402
                                     naive_bayes_input)

W_TOL, F_TOL, NB_TOL = 1e-9, 1e-11, 1e-12


@pytest.fixture(scope="module")
def ctx():
    import keystone_b200 as ks
    c = ks.Context(0)
    yield c
    c.close()


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


def _lr_weights(model):
    """The fitted W (d x (k-1)) from the model's d x k blocks, after checking the pivot column is zero."""
    W = np.concatenate(model.xs, 0)
    assert np.all(W[:, 0] == 0.0)
    return W[:, 1:]


def make_csr(rng, n, d, per_row, zipf=False, messy=False, long_rows=0, nonneg=False):
    """A scipy CSR matrix with Zipf(1.1) or uniform columns; messy: unsorted rows, repeated entries, every 7th row empty; long_rows:
    that many rows of 3 * 256 + 5 entries."""
    counts = rng.poisson(per_row, n)
    if messy:
        counts[::7] = 0
    if long_rows:
        counts[rng.choice(n, long_rows, replace=False)] = 3 * 256 + 5
    p = None
    if zipf:
        p = 1.0 / np.arange(1, d + 1) ** 1.1
        p /= p.sum()
    ind, dat = [], []
    for r in range(n):
        c = rng.choice(d, int(counts[r]), p=p) if p is not None else rng.integers(0, d, int(counts[r]))
        if messy and len(c) > 1:
            c = np.concatenate([c, c[:2]])
            rng.shuffle(c)
        elif not messy:
            c = np.sort(c)
        ind.append(c)
        v = rng.random(len(c)) * 2.0 if nonneg else rng.standard_normal(len(c))
        dat.append(v)
    indptr = np.concatenate([[0], np.cumsum([len(c) for c in ind])]).astype(np.int64)
    return sp.csr_matrix((np.concatenate(dat), np.concatenate(ind).astype(np.int32), indptr), shape=(n, d))


def _planted_labels(rng, A, k, scale):
    """Labels drawn from a planted softmax model over A, so the fit has signal."""
    W = rng.standard_normal((A.shape[1], k - 1)) * scale
    Z = np.hstack([np.zeros((A.shape[0], 1)), np.asarray(A @ W)])
    G = Z + rng.gumbel(size=Z.shape)
    return np.argmax(G, axis=1)


def _dense_case(rng, n, d, k):
    X = (rng.standard_normal((n, d)) * (2.0 / math.sqrt(d))).astype(np.float32)
    y = _planted_labels(rng, X.astype(np.float64), k, 1.0)
    return X, X.astype(np.float64), y


# ---------------------------------------------------------------------------------------------------------- 1. the suites
def test_binary_suite(ctx):
    """LogisticRegressionModelSuite 'logistic regression with LBFGS' through the nodes on dense device input."""
    import keystone_b200 as ks
    y, X = logistic_input(0.0, -0.8, 10000, 42)
    est = ks.LogisticRegressionEstimator(2, ctx=ctx)
    model = est.fit(ctx.matrix(X.astype(np.float32)), y)
    assert isinstance(model, ks.LogisticRegressionModel)
    assert model.num_classes == 2 and model.num_features == 1 and model.intercept == 0.0
    assert abs(model.weights[0] - (-0.8)) <= 0.03
    yv, Xv = logistic_input(0.0, -0.8, 10000, 17)
    pred = model.apply(ctx.matrix(Xv.astype(np.float32)))
    assert pred.dtype == np.float64 and (pred == yv).mean() > 0.65
    assert model.apply(Xv[0].astype(np.float32)) in (0.0, 1.0)
    assert est.stats["solver"] == "logistic_regression" and len(est.line_search_evals) >= est.iterations


def test_multinomial_suite(ctx):
    import keystone_b200 as ks
    y, X = multinomial_input(10000, 42)
    model = ks.LogisticRegressionEstimator(3, num_iters=200, convergence_tol=1e-15, ctx=ctx).fit(ctx.matrix(X.astype(np.float32)), y)
    assert np.abs(model.weights - MULTI_WEIGHTS_R).max() <= 0.05
    yv, Xv = multinomial_input(10000, 17)
    assert (model.apply(ctx.matrix(Xv.astype(np.float32))) == yv).mean() > 0.47


def test_naive_bayes_suite(ctx):
    import keystone_b200 as ks
    y, X = naive_bayes_input(1000, 42)
    model = ks.NaiveBayesEstimator(3, 1.0, ctx=ctx).fit(ctx.matrix(X.astype(np.float32)), y)
    assert isinstance(model, ks.NaiveBayesModel)
    assert np.abs(np.exp(model.pi) - NB_PI).max() <= 0.05
    assert np.abs(np.exp(model.theta) - NB_THETA).max() <= 0.05
    yv, Xv = naive_bayes_input(1000, 17)
    pred = ks.MaxClassifier().apply(model.apply(ctx.matrix(Xv.astype(np.float32))))
    assert (pred == yv).mean() >= 0.8


# ---------------------------------------------------------------------------------------------------------- 2. iterates
CASES = [  # input, n, d, k, lambda, iterations, sparse options
    ("dense", 3000, 1, 2, 0.0, 5, {}),
    ("dense", 3000, 4, 3, 1e-3, 8, {}),
    ("dense", 4000, 517, 20, 1e-3, 8, {}),
    ("dense", 2500, 4500, 3, 1e-3, 6, {}),
    ("sparse", 3000, 100003, 2, 1e-3, 6, dict(per_row=25, zipf=True, messy=True)),
    ("sparse", 2000, 517, 20, 0.0, 6, dict(per_row=12, messy=True, long_rows=3)),
    ("sparse", 2000, 4, 3, 0.1, 8, dict(per_row=2, messy=True)),
]


@pytest.mark.parametrize("kind,n,d,k,lam,iters,opts", CASES, ids=[f"{c[0]}-d{c[2]}-k{c[3]}-lam{c[4]}" for c in CASES])
def test_iterates_match_oracle(ctx, kind, n, d, k, lam, iters, opts):
    import keystone_b200 as ks
    rng = np.random.default_rng(d * 31 + k)
    if kind == "dense":
        X32, A, y = _dense_case(rng, n, d, k)
        data = ctx.matrix(X32)
    else:
        A = make_csr(rng, n, d, **opts)
        y = _planted_labels(rng, A, k, 1.0)
        data = ctx.sparse(A)
    est = ks.LogisticRegressionEstimator(k, reg_param=lam, num_iters=iters, convergence_tol=0.0, ctx=ctx)
    model = est.fit(data, y)
    W_ref, info = co.logistic_fit(A, y, k, reg_param=lam, num_iters=iters, convergence_tol=0.0)
    assert info["stop_reason"] == "max_iterations" and info["iterations"] == iters
    assert est.stop_reason == info["stop_reason"] and est.iterations == info["iterations"]
    assert est.line_search_evals == info["line_search_evals"]
    assert np.abs(np.array(est.loss_history) - info["loss_history"]).max() <= F_TOL * math.log(k)
    assert _rel(_lr_weights(model), W_ref) <= W_TOL
    assert est.stats["input"] == kind and est.stats["n_total"] == n
    # predictions: the oracle's fp64 rule, except where the two largest margins are closer than the apply path's rounding
    Z = np.hstack([np.zeros((n, 1)), np.asarray(A @ W_ref)])
    top = np.sort(Z, axis=1)
    clear = top[:, -1] - top[:, -2] > 1e-3 * (1.0 + np.abs(Z).max(1))
    pred = model.apply(data)
    assert np.array_equal(pred[clear], co.logistic_predict(W_ref, A)[clear])


def test_separable_data_stays_finite(ctx):
    import keystone_b200 as ks
    X = np.concatenate([np.linspace(0.5, 3, 500), -np.linspace(0.5, 3, 500)]).astype(np.float32)[:, None]
    y = np.array([1] * 500 + [0] * 500)
    est = ks.LogisticRegressionEstimator(2, num_iters=100, convergence_tol=0.0, ctx=ctx)
    model = est.fit(ctx.matrix(X), y)
    W = np.concatenate(model.xs, 0)
    assert np.isfinite(W).all() and np.isfinite(est.loss_history).all()
    assert (model.apply(ctx.matrix(X)) == y).all()


@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_refit_is_bit_identical(ctx, kind):
    import keystone_b200 as ks
    rng = np.random.default_rng(4)
    if kind == "dense":
        X32, A, y = _dense_case(rng, 5000, 700, 5)
        data = ctx.matrix(X32)
    else:
        A = make_csr(rng, 5000, 20000, per_row=30, zipf=True, messy=True, long_rows=2, nonneg=True)
        y = _planted_labels(rng, A, 5, 1.0)
        data = ctx.sparse(A)
    fits = []
    for _ in range(2):
        est = ks.LogisticRegressionEstimator(5, reg_param=1e-3, num_iters=10, convergence_tol=0.0, ctx=ctx)
        fits.append((np.concatenate(est.fit(data, y).xs, 0).copy(), est.loss_history))
    assert np.array_equal(fits[0][0], fits[1][0]) and fits[0][1] == fits[1][1]
    nb = [np.concatenate(ks.NaiveBayesEstimator(5, ctx=ctx).fit(data if kind == "sparse" else ctx.matrix(np.abs(X32)), y).xs, 0).copy()
          for _ in range(2)]
    assert np.array_equal(nb[0], nb[1])


# ---------------------------------------------------------------------------------------------------------- 3. naive Bayes
@pytest.mark.parametrize("kind,values", [("dense", "counts"), ("dense", "reals"), ("sparse", "counts"), ("sparse", "reals")])
def test_naive_bayes_matches_oracle(ctx, kind, values):
    import keystone_b200 as ks
    rng = np.random.default_rng(9)
    n, k = 3000, 7
    d = 5000 if kind == "dense" else 100003
    if kind == "dense":
        X = rng.poisson(0.3, (n, d)).astype(np.float64) if values == "counts" else rng.random((n, d)) * (rng.random((n, d)) < 0.2)
        X = X.astype(np.float32)
        A, data = X.astype(np.float64), ctx.matrix(X)
    else:
        A = make_csr(rng, n, d, per_row=40, zipf=True, messy=True, long_rows=2, nonneg=True)
        if values == "counts":
            A.data = np.ceil(A.data * 3)
        data = ctx.sparse(A)
    y = rng.integers(0, k, n)
    model = ks.NaiveBayesEstimator(k, 0.5, ctx=ctx).fit(data, y)
    pi, theta = co.naive_bayes_fit(A, y, k, 0.5)
    assert np.abs(model.pi - pi).max() <= NB_TOL * max(1.0, np.abs(pi).max())
    assert np.abs(model.theta - theta).max() <= NB_TOL * max(1.0, np.abs(theta).max())
    scores = model.apply(data).to_numpy()
    ref = np.asarray(A @ theta.T) + pi
    assert np.abs(scores - ref).max() <= 1e-4 * (1.0 + np.abs(ref).max())


def test_naive_bayes_model_from_host_and_save_load(ctx, tmp_path):
    import keystone_b200 as ks
    rng = np.random.default_rng(2)
    theta = np.log(rng.dirichlet(np.ones(6), 3))
    pi = np.log(np.array([0.2, 0.3, 0.5]))
    m = ks.NaiveBayesModel(np.array([0, 1, 2]), pi, theta, ctx=ctx)
    X = rng.poisson(1.0, (50, 6)).astype(np.float32)
    assert np.allclose(m.apply(ctx.matrix(X)).to_numpy(), X.astype(np.float64) @ theta.T + pi, rtol=1e-5, atol=1e-4)
    assert np.array_equal(m.pi, pi) and np.array_equal(m.theta, theta)
    path = str(tmp_path / "nb.ksb")
    m.save(path)
    m2 = ks.NaiveBayesModel.load(ctx, path)
    assert np.array_equal(m2.theta, theta) and np.array_equal(m2.pi, pi)
    y, Xl = logistic_input(0.0, -0.8, 2000, 42)
    lr = ks.LogisticRegressionEstimator(2, num_iters=5, ctx=ctx).fit(ctx.matrix(Xl.astype(np.float32)), y)
    lr.save(str(tmp_path / "lr.ksb"))
    lr2 = ks.LogisticRegressionModel.load(ctx, str(tmp_path / "lr.ksb"))
    assert np.array_equal(lr2.weights, lr.weights)
    assert np.array_equal(lr2.apply(ctx.matrix(Xl.astype(np.float32))), lr.apply(ctx.matrix(Xl.astype(np.float32))))


# ---------------------------------------------------------------------------------------------------------- 4. rejections
def test_abi_rejections(ctx):
    import keystone_b200 as ks
    from keystone_b200._capi import lib
    h = C.c_int64(0)
    dm = ctx.matrix(np.ones((4, 3), dtype=np.float32))
    sm = ctx.sparse(sp.csr_matrix(np.ones((4, 3))))
    y = np.array([0, 1, 1, 0], dtype=np.int32)
    yp = y.ctypes.data_as(C.c_void_p)
    lr = lambda f, s, yy, n, k, lam=0.0, it=10, tol=1e-4: lib().ks_logistic_fit(ctx.handle, f, s, yy, n, k, lam, it, tol, C.byref(h))  # noqa: E731
    nb = lambda f, s, yy, n, k, lam=1.0: lib().ks_naive_bayes_fit(ctx.handle, f, s, yy, n, k, lam, C.byref(h))  # noqa: E731
    assert lr(dm.handle, 0, yp, 4, 2) == 0 and nb(dm.handle, 0, yp, 4, 2) == 0
    assert lr(0, sm.handle, yp, 4, 2) == 0 and nb(0, sm.handle, yp, 4, 2) == 0
    for fn in (lr, nb):
        assert fn(dm.handle, sm.handle, yp, 4, 2) == -1          # two sources
        assert fn(0, 0, yp, 4, 2) == -1                          # none
        assert fn(dm.handle, 0, yp, 4, 1) == -1                  # num_classes < 2
        assert fn(dm.handle, 0, yp, 3, 2) == -1                  # n_labels != rows
        assert fn(0, dm.handle, yp, 4, 2) == -6                  # a dense handle as the sparse source
        assert fn(sm.handle, 0, yp, 4, 2) == -6                  # and the reverse
        bad = np.array([0, 1, 2, 0], dtype=np.int32)
        assert fn(dm.handle, 0, bad.ctypes.data_as(C.c_void_p), 4, 2) == -1   # label outside [0, k)
        neg = np.array([0, 1, -1, 0], dtype=np.int32)
        assert fn(dm.handle, 0, neg.ctypes.data_as(C.c_void_p), 4, 2) == -1
        assert "numClasses" in lib().ks_last_error(ctx.handle).decode()
    for kw in [(-1.0, 10, 1e-4), (float("nan"), 10, 1e-4), (0.0, 0, 1e-4), (0.0, 10, -1.0), (0.0, 10, float("inf"))]:
        assert lr(dm.handle, 0, yp, 4, 2, *kw) == -1, kw
    assert nb(dm.handle, 0, yp, 4, 2, -1.0) == -1 and nb(dm.handle, 0, yp, 4, 2, float("nan")) == -1
    assert nb(dm.handle, 0, yp, 4, 3) == -1                      # class 2 has no rows
    assert "no training rows" in lib().ks_last_error(ctx.handle).decode()
    dneg = ctx.matrix(np.array([[1, 0, 0], [0, -1, 0], [1, 1, 1], [0, 0, 2]], dtype=np.float32))
    sneg = ctx.sparse(sp.csr_matrix(np.array([[1.0, 0, 0], [0, -1, 0], [1, 1, 1], [0, 0, 2]])))
    assert nb(dneg.handle, 0, yp, 4, 2) == -1 and nb(0, sneg.handle, yp, 4, 2) == -1
    assert "negative" in lib().ks_last_error(ctx.handle).decode()
    dnan = ctx.matrix(np.array([[1, 0, 0], [0, np.nan, 0], [1, 1, 1], [0, 0, 2]], dtype=np.float32))
    assert nb(dnan.handle, 0, yp, 4, 2) == -1
    assert lib().ks_logistic_fit(ctx.handle, dm.handle, 0, yp, 4, 2, 0.0, 10, 1e-4, None) == -1
    # the nodes
    with pytest.raises(ks.KeystoneError, match="num_features"):
        ks.LogisticRegressionEstimator(2, num_features=5, ctx=ctx).fit(dm, y)
    x_in = ctx.matrix(np.ones((4, 2), dtype=np.float32))
    lazy = ks.CosineRandomFeatures(ctx, np.ones((3, 2), dtype=np.float32), np.zeros(3, dtype=np.float32)).apply(x_in)
    with pytest.raises(ks.KeystoneError, match="LazyFeatures"):
        ks.LogisticRegressionEstimator(2, ctx=ctx).fit(lazy, y)
    with pytest.raises(ks.KeystoneError, match="LazyFeatures"):
        ks.NaiveBayesEstimator(2, ctx=ctx).fit(lazy, y)
    with pytest.raises(ValueError):
        ks.LogisticRegressionEstimator(1)
    with pytest.raises(ValueError):
        ks.NaiveBayesEstimator(2, lam=-1.0)


# ---------------------------------------------------------------------------------------------------------- 5. two ranks
def _worker(rank, world, id_holder, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import keystone_b200 as ks
    rng = np.random.default_rng(8)
    n, d, k = 3001, 4500, 3
    A = make_csr(rng, n, d, per_row=30, zipf=True, messy=True, long_rows=3, nonneg=True)
    y = _planted_labels(rng, A, k, 1.0)
    X32 = np.asarray(A[:, :300].todense(), dtype=np.float32)
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    for name, split in (("uneven", 1000), ("empty", n)):   # rank 1 holds rows [split, n): none in the second fit
        r0, r1 = (0, split) if rank == 0 else (split, n)
        for kind, data in (("sparse", ctx.sparse(A[r0:r1])), ("dense", ctx.matrix(X32[r0:r1]))):
            est = ks.LogisticRegressionEstimator(k, reg_param=0.01, num_iters=8, convergence_tol=0.0, ctx=ctx)
            m = est.fit(data, y[r0:r1])
            ret[f"{name}{kind}W{rank}"] = np.concatenate(m.xs, 0).copy()
            ret[f"{name}{kind}loss{rank}"] = est.loss_history
            ret[f"{name}{kind}NB{rank}"] = np.concatenate(ks.NaiveBayesEstimator(k, ctx=ctx).fit(data, y[r0:r1]).xs, 0).copy()
    # a bad label on rank 1 only: both ranks reject the fit
    yb = y[1000:].copy() if rank == 1 else y[:1000]
    if rank == 1:
        yb[5] = k
    data = ctx.sparse(A[:1000] if rank == 0 else A[1000:])
    for est in (ks.LogisticRegressionEstimator(k, num_iters=3, ctx=ctx), ks.NaiveBayesEstimator(k, ctx=ctx)):
        try:
            est.fit(data, yb)
            ret[f"bad{type(est).__name__}{rank}"] = "fitted"
        except ks.KeystoneError as e:
            ret[f"bad{type(est).__name__}{rank}"] = str(e)
    ctx.close()
    if rank == 0:
        c1 = ks.Context(device=0)
        for kind, data in (("sparse", c1.sparse(A)), ("dense", c1.matrix(X32))):
            e1 = ks.LogisticRegressionEstimator(k, reg_param=0.01, num_iters=8, convergence_tol=0.0, ctx=c1)
            ret[f"{kind}W1rank"] = np.concatenate(e1.fit(data, y).xs, 0).copy()
            ret[f"{kind}loss1rank"] = e1.loss_history
            ret[f"{kind}NB1rank"] = np.concatenate(ks.NaiveBayesEstimator(k, ctx=c1).fit(data, y).xs, 0).copy()
        c1.close()


def test_two_ranks_equal_one_rank():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import keystone_b200 as ks
    mgr = mp.Manager()
    id_holder = mgr.dict(); ret = mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    for name in ("uneven", "empty"):
        for kind in ("sparse", "dense"):
            assert np.array_equal(ret[f"{name}{kind}W0"], ret[f"{name}{kind}W1"])
            assert ret[f"{name}{kind}loss0"] == ret[f"{name}{kind}loss1"]
            assert np.array_equal(ret[f"{name}{kind}NB0"], ret[f"{name}{kind}NB1"])
            assert _rel(ret[f"{name}{kind}W0"], ret[f"{kind}W1rank"]) <= 1e-9
            assert _rel(ret[f"{name}{kind}NB0"], ret[f"{kind}NB1rank"]) <= 1e-12
    for est in ("LogisticRegressionEstimator", "NaiveBayesEstimator"):
        assert "numClasses" in ret[f"bad{est}0"] and "numClasses" in ret[f"bad{est}1"]
