"""Gaussian-kernel ridge regression on the H100 through the C ABI / node API, against the fp64 oracle (tests/krr_oracle.py).

Gates follow from the operand precision: every MMA operand is an fp16 pair (>= 21 significant bits) and the fitted systems are
kept at cond(K + lambda I) <= 100, so W is expected within ~1e-4 relative of the fp64 oracle.  Inputs are uploaded as fp32 (the
library's matrix format), so the oracle is evaluated on the fp32-rounded inputs."""
import ctypes as C
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
import krr_oracle as ko  # noqa: E402


@pytest.fixture(scope="module")
def ctx():
    import keystone_b200 as ks
    c = ks.Context(0)
    yield c
    c.close()


def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _kernel_exact(X, Z, gamma):
    """exp(-gamma |x - z|^2) from the differences (no cancellation): the reference values of the offset data."""
    X, Z = _f32(X), _f32(Z)
    d2 = ((X[:, None, :] - Z[None, :, :]) ** 2).sum(-1) if X.shape[0] * Z.shape[0] * X.shape[1] < 3e7 else None
    if d2 is None:
        m = X.mean(0)
        Xc, Zc = X - m, Z - m
        d2 = (Xc ** 2).sum(1)[:, None] + (Zc ** 2).sum(1)[None, :] - 2 * Xc @ Zc.T
    return np.exp(-gamma * d2)


# ---------------------------------------------------------------------------------------------------------- 1. kernel block
@pytest.mark.parametrize("n,d,cols,col0", [(1, 1, 1, 0), (127, 2, 37, 90), (1000, 37, 300, 0), (1000, 37, 300, 700),
                                           (4097, 440, 500, 3597), (4097, 1, 37, 10), (127, 440, 1, 126)])
@pytest.mark.parametrize("offset", [0.0, 100.0])
def test_kernel_block_matches_oracle(ctx, n, d, cols, col0, offset):
    import keystone_b200 as ks
    rng = np.random.default_rng(n * 7 + d)
    gamma = 2.0 / (2 * d)                          # gamma |x - m|^2 ~ 1, <= ~4 over the sample
    X = rng.standard_normal((n, d)) + offset
    T = rng.standard_normal((200, d)) + offset
    tr = ks.GaussianKernelGenerator(gamma, ctx=ctx).fit(X.astype(np.float32))
    assert tr.n_train == n and tr.dim == d
    km = tr.apply(T.astype(np.float32))
    got = km(range(col0, col0 + cols)).to_numpy()
    ref = _kernel_exact(T, X[col0:col0 + cols], gamma)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 2e-5
    # diag_block: K(rows idxs of the dataset, training rows idxs), here with the training rows as the dataset
    if col0 + cols <= n:
        kd = tr.apply(X.astype(np.float32)).diag_block(range(col0, col0 + cols))
        assert np.abs(kd - _kernel_exact(X[col0:col0 + cols], X[col0:col0 + cols], gamma)).max() <= 2e-5


def test_kernel_row_of_a_vector(ctx):
    import keystone_b200 as ks
    rng = np.random.default_rng(1)
    X = rng.standard_normal((300, 8))
    tr = ks.GaussianKernelGenerator(0.1, ctx=ctx).fit(X.astype(np.float32))
    row = tr.apply(X[5])
    assert row.shape == (300,)
    assert np.abs(row - _kernel_exact(X[5:6], X, 0.1)[0]).max() <= 2e-5


# ---------------------------------------------------------------------------------------------------------- 2. XOR
@pytest.mark.parametrize("block_size", [4, 2])
def test_xor_known_answer(ctx, block_size):
    """KernelModelSuite's two XOR cases: gamma 10, lambda 0, 2 epochs."""
    import keystone_b200 as ks
    x = np.array([[-1.0, -1.0], [1.0, 1.0], [-1.0, 1.0], [1.0, -1.0]])
    y = np.array([[0.0, 1.0], [0.0, 1.0], [1.0, 0.0], [1.0, 0.0]])
    model = ks.KernelRidgeRegression(ks.GaussianKernelGenerator(10.0), 0.0, block_size, 2, ctx=ctx).fit(ctx.matrix(x), ctx.matrix(y))
    pred = model.apply(ctx.matrix(x[:3])).to_numpy()
    assert np.sum((pred - y[:3]) ** 2) < 1e-4


# ---------------------------------------------------------------------------------------------------------- 3. / 4. fit parity
def _parity_problem(scale_late=False):
    rng = np.random.default_rng(11)
    n, d, k, n_test = 2300, 40, 6, 500
    X = _f32(rng.standard_normal((n + n_test, d)))
    cls = rng.integers(0, k, n + n_test)
    Y = -np.ones((n + n_test, k))
    Y[np.arange(n + n_test), cls] = 1.0
    if scale_late:
        Y[1000:n] *= 1000.0                        # later blocks force a larger operand exponent of W mid-fit
    gamma = 1.0 / d
    K = ko.gaussian_kernel(X[:n], X[:n], gamma)
    ev = np.linalg.eigvalsh(K)
    lam = float(ev[-1] / 99.0)
    cond = (ev[-1] + lam) / (ev[0] + lam)
    assert cond <= 100.0, cond
    return X[:n], Y[:n], X[n:], gamma, lam


@pytest.mark.parametrize("permuted", [False, True], ids=["sequential", "permuted"])
@pytest.mark.parametrize("scale_late", [False, True], ids=["plain", "operand-rescale"])
def test_fit_matches_oracle(ctx, permuted, scale_late):
    import keystone_b200 as ks
    X, Y, Xt, gamma, lam = _parity_problem(scale_late)
    bs, epochs = 500, 2                            # not a multiple of 32; 300-row ragged tail
    est = ks.KernelRidgeRegression(ks.GaussianKernelGenerator(gamma), lam, bs, epochs, block_permuter=3 if permuted else None, ctx=ctx)
    model = est.fit(ctx.matrix(X.astype(np.float32)), ctx.matrix(Y.astype(np.float32)))
    st = ctx.last_fit_stats()
    assert st["solver"] == "krr" and st["num_blocks"] == 5 and st["mma"] == "f16x2"
    for key in ("generate_ms", "gram_ms", "solve_ms", "update_ms", "total_ms"):
        assert st[key] >= 0.0
    order = est.block_order(len(X))
    xs_ref = ko.krr_fit(X, Y, gamma, lam, bs, epochs, None if order is None else order.tolist())
    W, Wr = np.concatenate(model.xs, 0), np.concatenate(xs_ref, 0)
    assert [w.shape[0] for w in model.xs] == [500, 500, 500, 500, 300]
    rel = np.linalg.norm(W - Wr) / np.linalg.norm(Wr)
    assert rel <= 1e-4, rel
    pred = model.apply(ctx.matrix(Xt.astype(np.float32))).to_numpy()
    pref = ko.kernel_block_apply(Xt, X, gamma, xs_ref, bs)
    assert np.abs(pred - pref).max() <= 1e-4 * np.abs(Y).max()
    assert np.array_equal(model.apply_argmax(ctx.matrix(Xt.astype(np.float32))), np.argmax(pred.astype(np.float32), 1))


# ---------------------------------------------------------------------------------------------------------- 5. apply alone
def test_apply_from_arrays_matches_oracle(ctx):
    import keystone_b200 as ks
    rng = np.random.default_rng(5)
    X = _f32(rng.standard_normal((777, 13)) * 2 + 5)
    Xt = _f32(rng.standard_normal((333, 13)) * 2 + 5)
    gamma, bs = 0.02, 256
    xs = [rng.standard_normal((hi - lo, 4)) for lo, hi in ko.block_ranges(777, bs)]
    tr = ks.GaussianKernelGenerator(gamma, ctx=ctx).fit(X.astype(np.float32))
    model = ks.KernelBlockLinearMapper.from_arrays(ctx, xs, bs, tr)
    got = model.apply(ctx.matrix(Xt.astype(np.float32))).to_numpy()
    ref = ko.kernel_block_apply(Xt, X, gamma, xs, bs)
    assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max()
    with pytest.raises(ks.KeystoneError):        # block rows must sum to the training rows
        ks.KernelBlockLinearMapper.from_arrays(ctx, xs[:-1], bs, tr)


# ---------------------------------------------------------------------------------------------------------- 6. rejections
def test_rejections(ctx, tmp_path):
    import keystone_b200 as ks
    from keystone_b200._capi import lib
    rng = np.random.default_rng(2)
    X = rng.standard_normal((40, 3)).astype(np.float32)
    Y = rng.standard_normal((40, 2)).astype(np.float32)
    x, y = ctx.matrix(X), ctx.matrix(Y)
    model = ks.KernelRidgeRegression(ks.GaussianKernelGenerator(0.5), 0.1, 16, 1, ctx=ctx).fit(x, y)
    L, h, cost = lib(), C.c_int64(0), C.c_double(0)

    def invalid(rc):
        assert rc == -1, rc
        assert ctx and L.ks_last_error(ctx.handle)

    invalid(L.ks_model_save(ctx.handle, model.handle, str(tmp_path / "m.bin").encode()))
    invalid(L.ks_model_cost(ctx.handle, model.handle, x.handle, 0, None, 0, y.handle, 0.1, C.byref(cost)))
    invalid(L.ks_model_apply_partial(ctx.handle, model.handle, x.handle, 0, None, 0, 0, C.byref(h)))
    invalid(L.ks_model_apply(ctx.handle, model.handle, x.handle, x.handle, None, 0, C.byref(h)))          # x_in given
    rf = ks.CosineRandomFeatures(ctx, rng.standard_normal((8, 3)), rng.standard_normal(8))
    rfs = (C.c_int64 * 1)(rf.handle)
    invalid(L.ks_model_apply(ctx.handle, model.handle, 0, x.handle, rfs, 1, C.byref(h)))                # rfs given
    x2, y30 = ctx.matrix(X[:, :2]), ctx.matrix(Y[:30])
    invalid(L.ks_model_apply(ctx.handle, model.handle, x2.handle, 0, None, 0, C.byref(h)))                # column count
    kern = model.kernel_transformer.handle
    bad = np.array([[0, 0, 1]], dtype=np.int32)                                                       # not a permutation
    invalid(L.ks_krr_fit(ctx.handle, kern, y.handle, 0.1, 16, 1, bad.ctypes.data_as(C.c_void_p), C.byref(h)))
    invalid(L.ks_krr_fit(ctx.handle, kern, y.handle, 0.1, 0, 1, None, C.byref(h)))                    # block_size < 1
    invalid(L.ks_krr_fit(ctx.handle, kern, y.handle, 0.1, 16, 0, None, C.byref(h)))                   # num_epochs < 1
    invalid(L.ks_krr_fit(ctx.handle, kern, y30.handle, 0.1, 16, 1, None, C.byref(h)))                # label rows
    invalid(L.ks_gaussian_kernel_create(ctx.handle, x.handle, 0.0, C.byref(h)))
    invalid(L.ks_gaussian_kernel_create(ctx.handle, x.handle, float("nan"), C.byref(h)))
    invalid(L.ks_gaussian_kernel_block(ctx.handle, kern, x.handle, 30, 11, C.byref(h)))                # past the last column
    # lambda = 0 with a repeated training row: K_BB + lambda I is singular
    Xd = np.concatenate([X[:10], X[:1]], 0)
    with pytest.raises(ks.KeystoneError) as ei:
        ks.KernelRidgeRegression(ks.GaussianKernelGenerator(0.5), 0.0, 16, 1, ctx=ctx).fit(ctx.matrix(Xd), ctx.matrix(Y[:11]))
    assert ei.value.code == -7
    # the context is still usable
    assert model.apply(x).to_numpy().shape == (40, 2)


# ---------------------------------------------------------------------------------------------------------- 7. two ranks
def _two_rank_worker(rank, world, id_holder, ret):
    sys.path.insert(0, ROOT)
    import keystone_b200 as ks
    rng = np.random.default_rng(31)
    n, d, k = 6001, 20, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    Xt = rng.standard_normal((400, d)).astype(np.float32)
    Y = rng.standard_normal((n, k)).astype(np.float32)
    lo, hi = (0, 3000) if rank == 0 else (3000, n)     # block 5 ([2560, 3072)) straddles the ranks
    tlo, thi = (0, 150) if rank == 0 else (150, 400)
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    model = ks.KernelRidgeRegression(ks.GaussianKernelGenerator(1.0 / d), 2.0, 512, 2, ctx=ctx).fit(ctx.matrix(X[lo:hi]),
                                                                                                     ctx.matrix(Y[lo:hi]))
    ret[f"W{rank}"] = np.concatenate(model.xs, 0).copy()
    ret[f"P{rank}"] = model.apply(ctx.matrix(Xt[tlo:thi])).to_numpy()
    ctx.close()


def test_two_rank_fit_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import keystone_b200 as ks
    mgr = mp.Manager()
    id_holder, ret = mgr.dict(), mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_two_rank_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    rng = np.random.default_rng(31)
    n, d, k = 6001, 20, 5
    X = _f32(rng.standard_normal((n, d)))
    Xt = _f32(rng.standard_normal((400, d)))
    Y = _f32(rng.standard_normal((n, k)))
    xs = ko.krr_fit(X, Y, 1.0 / d, 2.0, 512, 2)
    Wr = np.concatenate(xs, 0)
    assert np.array_equal(ret["W0"], ret["W1"])
    assert np.linalg.norm(ret["W0"] - Wr) / np.linalg.norm(Wr) <= 1e-4
    P = np.concatenate([ret["P0"], ret["P1"]], 0)
    assert np.abs(P - ko.kernel_block_apply(Xt, X, 1.0 / d, xs, 512)).max() <= 1e-4 * np.abs(Y).max()
