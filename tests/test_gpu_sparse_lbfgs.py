"""Sparse L-BFGS least squares (SparseLBFGSwithL2), SparseLinearMapper and Densify on the H100, against the fp64 oracle: the dense
L-BFGS oracle (tests/lbfgs_oracle.py) on [A 1] with fp32-rounded labels (DESIGN.md section 20).

Everything after the labels is fp64 on both sides, so only summation order differs: rel-Frobenius([W; b]) <= 1e-9 and loss history
<= 1e-11 relative to f(x_0).  Every fitted problem has cond([A 1]^T [A 1] / N + lambda I) <= 100."""
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
import lbfgs_oracle as lo  # noqa: E402
from test_oracle_sparse_lbfgs import DATA_MEAN, EXTRA_BIAS, X_TRUE, sparse_suite_data  # noqa: E402

W_TOL, F_TOL = 1e-9, 1e-11


@pytest.fixture(scope="module")
def ctx():
    import keystone_b200 as ks
    c = ks.Context(0)
    yield c
    c.close()


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


def _csr_from_dense(A):
    rows, cols = np.nonzero(A)
    indptr = np.zeros(A.shape[0] + 1, dtype=np.int64)
    np.add.at(indptr, rows + 1, 1)
    return np.cumsum(indptr), cols.astype(np.int32), A[rows, cols]


def make_sparse(rng, n, d, per_row, zipf=False, full_col=False, messy=False, long_rows=0):
    """(indptr, indices, data) and the dense fp64 matrix with repeated entries summed.  zipf: Zipf(1.1) column popularity;
    full_col: column 0 in every row; messy: unsorted rows, repeated (row, column) entries, every 7th row empty, the last
    column empty; long_rows: that many rows with 3 * 256 + 5 entries (split into several chunks)."""
    counts = rng.poisson(per_row, n).clip(0, d)
    if messy:
        counts[::7] = 0
    if long_rows:
        counts[rng.choice(n, long_rows, replace=False)] = min(3 * 256 + 5, 4 * d)
    if zipf:
        p = 1.0 / np.arange(1, d + 1) ** 1.1
        p /= p.sum()
    ind, dat = [], []
    for r in range(n):
        cnt = int(counts[r])
        if cnt == 0 and not (full_col and not (messy and r % 7 == 0)):
            ind.append(np.zeros(0, np.int64)); dat.append(np.zeros(0)); continue
        c = rng.choice(d, cnt, p=p) if zipf else rng.integers(0, d, cnt)
        if messy:
            c = c[c != d - 1] if d > 1 else c
            if len(c) > 1:
                c = np.concatenate([c, c[:2]])       # repeated entries
            rng.shuffle(c)                           # unsorted
        else:
            c = np.sort(c)
        if full_col and not (messy and r % 7 == 0):
            c = np.concatenate([[0], c])
        ind.append(c); dat.append(rng.standard_normal(len(c)))
    indptr = np.concatenate([[0], np.cumsum([len(c) for c in ind])]).astype(np.int64)
    indices = np.concatenate(ind).astype(np.int32)
    data = np.concatenate(dat)
    A = np.zeros((n, d))
    np.add.at(A, (np.repeat(np.arange(n), np.diff(indptr)), indices), data)
    return (indptr, indices, data), A


def _augment(A, fit_intercept):
    return np.hstack([A, np.ones((A.shape[0], 1))]) if fit_intercept else A


def _lam_for_cond(Aug, cond=99.0):
    n, D = Aug.shape
    G = Aug @ Aug.T / n if n < D else Aug.T @ Aug / n
    ev = np.linalg.eigvalsh(G)
    lo_ev = 0.0 if n < D else ev[0]
    return max(0.0, (ev[-1] - cond * lo_ev) / (cond - 1.0)) + 1e-12


def _model_x(mapper, fit_intercept):
    W = np.concatenate(mapper.xs, 0)
    return np.vstack([W, mapper.b_opt[None, :]]) if fit_intercept else W


# ---------------------------------------------------------------------------------------------------------- 1. known answers
@pytest.mark.parametrize("fit_intercept,tol", [(True, 1e-3), (False, 1e-4)])
def test_suite_known_answers(ctx, fit_intercept, tol):
    """LBFGSSuite.scala:62-108 through the node at the default parameters and the suite's tolerances."""
    import keystone_b200 as ks
    A, B = sparse_suite_data(fit_intercept)
    sm = ctx.sparse(_csr_from_dense(A) + (A.shape[1],))
    est = ks.SparseLBFGSwithL2(ks.LeastSquaresSparseGradient(), fit_intercept=fit_intercept, ctx=ctx)
    mapper = est.fit(sm, B.astype(np.float32))
    assert isinstance(mapper, ks.SparseLinearMapper)
    assert np.abs(mapper.apply(sm).to_numpy() - B).max() < tol
    assert np.abs(mapper.x - X_TRUE.T).max() < tol
    if fit_intercept:
        assert np.abs(mapper.b_opt - (EXTRA_BIAS - X_TRUE @ DATA_MEAN)).max() < tol
    else:
        assert mapper.b_opt is None
    assert mapper.feature_means is None
    assert est.stats["solver"] == "sparse_lbfgs" and est.stats["nnz"] == np.count_nonzero(A)
    assert est.iterations >= 1 and len(est.loss_history) == est.iterations + 1


# ---------------------------------------------------------------------------------------------------------- 2. iterates
CASES = [  # n, d, k, fit_intercept, options of make_sparse (d = 1 with an intercept: 2 unknowns, solved exactly by step 2)
    (2000, 1, 1, True, dict(per_row=0.7, steps=2)),
    (3000, 517, 2, False, dict(per_row=12, zipf=True, full_col=True, messy=True, long_rows=3)),
    (3000, 1531, 20, True, dict(per_row=20, zipf=True, full_col=True, messy=True, long_rows=2)),
    (1200, 777, 147, True, dict(per_row=15, zipf=True, full_col=True, messy=True, long_rows=2)),
    (1500, 4500, 3, False, dict(per_row=30, zipf=True, messy=True)),
    (300, 100003, 2, True, dict(per_row=50, zipf=True, full_col=True)),
]


@pytest.mark.parametrize("n,d,k,fit_intercept,opts", CASES)
def test_iterates_match_oracle(ctx, n, d, k, fit_intercept, opts):
    """8 steps (2 at d = 1) with convergence_tol = 0 against the oracle on [A 1] with the same fp32-rounded labels."""
    import keystone_b200 as ks
    rng = np.random.default_rng(n + d + k)
    opts = dict(opts)
    steps = opts.pop("steps", 8)
    csr, A = make_sparse(rng, n, d, **opts)
    Aug = _augment(A, fit_intercept)
    Xt = rng.standard_normal((Aug.shape[1], k)) / np.sqrt(1 + opts["per_row"])
    Y = (Aug @ Xt + 0.3 * rng.standard_normal((n, k))).astype(np.float32)
    lam = _lam_for_cond(Aug)
    sm = ctx.sparse(csr + (d,))
    est = ks.SparseLBFGSwithL2(fit_intercept=fit_intercept, num_corrections=5, convergence_tol=0.0, num_iterations=steps,
                               reg_param=lam, ctx=ctx)
    mapper = est.fit(sm, Y)
    X, _, _, info = lo.fit(Aug, Y.astype(np.float64), False, 5, 0.0, steps, lam)
    assert est.iterations == steps and est.stop_reason == "max_iterations"
    assert est.stats["nnz"] == len(csr[1]) and est.stats["d"] == d
    assert [b.shape[0] for b in mapper.xs] == [min(4096, d - j) for j in range(0, d, 4096)]
    Xg = _model_x(mapper, fit_intercept)
    assert _rel(Xg, X) <= W_TOL, _rel(Xg, X)
    lh, ref = np.array(est.loss_history), np.array(info["loss_history"])
    assert np.abs(lh - ref).max() / np.abs(ref).max() <= F_TOL, np.abs(lh - ref).max() / np.abs(ref).max()


# ---------------------------------------------------------------------------------------------------------- 3. determinism
def test_repeated_fit_is_bit_identical(ctx):
    import keystone_b200 as ks
    rng = np.random.default_rng(21)
    csr, A = make_sparse(rng, 5000, 2000, per_row=25, zipf=True, full_col=True, messy=True, long_rows=4)
    Y = (A[:, :50] @ rng.standard_normal((50, 5)) + rng.standard_normal((5000, 5))).astype(np.float32)
    sm = ctx.sparse(csr + (2000,))
    fits = []
    for _ in range(2):
        est = ks.SparseLBFGSwithL2(num_iterations=12, convergence_tol=0.0, reg_param=1e-3, ctx=ctx)
        m = est.fit(sm, Y)
        fits.append((np.concatenate(m.xs, 0).copy(), m.b_opt.copy(), est.loss_history))
    assert np.array_equal(fits[0][0], fits[1][0]) and np.array_equal(fits[0][1], fits[1][1])
    assert fits[0][2] == fits[1][2]


# ---------------------------------------------------------------------------------------------------------- 4. the model, Densify
def test_apply_persistence_and_densify(ctx, tmp_path):
    import keystone_b200 as ks
    rng = np.random.default_rng(5)
    n, d, k = 3000, 1200, 4
    csr, A = make_sparse(rng, n, d, per_row=20, zipf=True, full_col=True, messy=True, long_rows=2)
    Y = (A @ rng.standard_normal((d, k)) * 0.1 + 1.0).astype(np.float32)
    sm = ctx.sparse(csr + (d,))
    m = ks.SparseLBFGSwithL2(num_iterations=10, reg_param=1e-2, ctx=ctx).fit(sm, Y)
    W, b = m.x.copy(), m.b_opt.copy()
    pred = m.apply(sm).to_numpy(np.float32)
    ref = (A @ W + b).astype(np.float32)
    assert np.all(np.abs(pred.astype(np.float64) - ref) <= np.spacing(np.abs(ref))), "A W + b rounded once to fp32"
    m2 = ks.SparseLinearMapper(W, b, ctx=ctx)   # from host arrays
    assert np.array_equal(m2.apply(sm).to_numpy(np.float32), pred)
    path = str(tmp_path / "sparse.ksm")
    m.save(path)
    m3 = ks.SparseLinearMapper.load(ctx, path)
    assert np.array_equal(m3.x, W) and np.array_equal(m3.b_opt, b) and m3.feature_means is None
    assert np.array_equal(m3.apply(sm).to_numpy(np.float32), pred)
    dense = ks.Densify().apply(sm)
    assert np.array_equal(dense.to_numpy(np.float32), A.astype(np.float32)), "Densify: repeated entries summed, rounded once"
    pd = ks.BlockLinearMapper.apply(m, dense).to_numpy()       # the dense ks_model_apply on Densify(A)
    assert np.abs(pd - ref).max() <= 1e-5 * np.abs(ref).max()
    # no intercept: A W alone
    m4 = ks.SparseLinearMapper(W, None, ctx=ctx)
    ref4 = (A @ W).astype(np.float32)
    assert np.all(np.abs(m4.apply(sm).to_numpy(np.float32).astype(np.float64) - ref4) <= np.spacing(np.abs(ref4)))


# ---------------------------------------------------------------------------------------------------------- 5. LeastSquaresEstimator
def test_least_squares_estimator_routes_sparse_input(ctx):
    import keystone_b200 as ks
    rng = np.random.default_rng(9)
    n, d, k = 3000, 10000, 2
    csr, A = make_sparse(rng, n, d, per_row=50, zipf=True)
    Y = (A[:, :100] @ rng.standard_normal((100, k)) + 0.1 * rng.standard_normal((n, k))).astype(np.float32)
    sm = ctx.sparse(csr + (d,))
    lam = 1e-3
    est = ks.LeastSquaresEstimator(lam=lam, ctx=ctx)
    m = est.fit(sm, Y)
    assert est.selected == "sparse_lbfgs" and est.used == "sparse_lbfgs"
    ref = ks.SparseLBFGSwithL2(num_iterations=20, reg_param=lam, ctx=ctx).fit(sm, Y)
    assert np.array_equal(np.concatenate(m.xs, 0), np.concatenate(ref.xs, 0)) and np.array_equal(m.b_opt, ref.b_opt)
    # small d: the exact solver on the densified matrix
    csr2, A2 = make_sparse(rng, 500, 20, per_row=6)
    Y2 = (A2 @ rng.standard_normal((20, 3)) + 0.1 * rng.standard_normal((500, 3))).astype(np.float32)
    sm2 = ctx.sparse(csr2 + (20,))
    est2 = ks.LeastSquaresEstimator(lam=0.5, ctx=ctx)
    m2 = est2.fit(sm2, Y2)
    assert est2.selected == "exact" and est2.used == "exact"
    ref2 = ks.LinearMapEstimator(0.5, ctx).fit(ctx.matrix(A2.astype(np.float32)), ctx.matrix(Y2))
    assert _rel(m2.x, ref2.x) <= 1e-5 and np.abs(m2.b_opt - ref2.b_opt).max() <= 1e-5 * np.abs(ref2.b_opt).max()


# ---------------------------------------------------------------------------------------------------------- 6. rejections
def test_rejections(ctx):
    import keystone_b200 as ks
    from keystone_b200._capi import lib
    h = C.c_int64(0)

    def up(indptr, indices, data, n_cols):
        ip = np.ascontiguousarray(indptr, dtype=np.int64)
        ix = np.ascontiguousarray(indices, dtype=np.int32)
        dv = np.ascontiguousarray(data, dtype=np.float64)
        return lib().ks_sparse_from_host_csr(ctx.handle, ip.ctypes.data_as(C.c_void_p), ix.ctypes.data_as(C.c_void_p),
                                             dv.ctypes.data_as(C.c_void_p), len(ip) - 1, n_cols, C.byref(h))

    good = ([0, 2, 2, 3], [1, 0, 2], [1.0, 2.0, 3.0], 3)
    assert up(*good) == 0
    lib().ks_sparse_destroy(ctx.handle, h.value)
    bad = [([1, 2, 2, 3], [1, 0, 2], [1.0, 2.0, 3.0], 3),            # indptr[0] != 0
           ([0, 2, 1, 3], [1, 0, 2], [1.0, 2.0, 3.0], 3),            # decreasing
           ([0, 2, 2, 3], [1, 0, 3], [1.0, 2.0, 3.0], 3),            # index >= n_cols
           ([0, 2, 2, 3], [1, -1, 2], [1.0, 2.0, 3.0], 3),           # negative index
           ([0, 2, 2, 3], [1, 0, 2], [1.0, np.nan, 3.0], 3),         # non-finite
           ([0, 2, 2, 3], [1, 0, 2], [1.0, 2.0, np.inf], 3),
           ([0, 0], [], [], 0),                                      # n_cols < 1
           ([0, 0], [], [], 2 ** 31)]                                # n_cols > INT32_MAX
    for args in bad:
        assert up(*args) == -1, args
        assert lib().ks_last_error(ctx.handle)
    with pytest.raises(ks.KeystoneError):                                # indptr[n_rows] != nnz
        ctx.sparse((np.array([0, 2, 4]), np.array([0, 1, 0]), np.ones(3), 2))

    sm = ctx.sparse(good)
    dm = ctx.matrix(np.ones((3, 3), dtype=np.float32))
    y = ctx.matrix(np.ones((3, 2), dtype=np.float32))
    y_bad = ctx.matrix(np.ones((4, 2), dtype=np.float32))
    # handles of the wrong type, both directions
    assert lib().ks_sparse_densify(ctx.handle, dm.handle, C.byref(h)) == -6
    assert lib().ks_sparse_lbfgs_fit(ctx.handle, dm.handle, y.handle, 1, 10, 1e-4, 10, 0.0, C.byref(h)) == -6
    assert lib().ks_sparse_lbfgs_fit(ctx.handle, sm.handle, sm.handle, 1, 10, 1e-4, 10, 0.0, C.byref(h)) == -6
    dense_model = ks.LinearMapper.from_arrays(ctx, np.ones((3, 2)), np.zeros(2))
    assert lib().ks_model_apply(ctx.handle, dense_model.handle, sm.handle, 0, None, 0, C.byref(h)) == -6
    assert lib().ks_model_apply_sparse(ctx.handle, dense_model.handle, dm.handle, C.byref(h)) == -6
    # rows of labels and data, model and data d
    assert lib().ks_sparse_lbfgs_fit(ctx.handle, sm.handle, y_bad.handle, 1, 10, 1e-4, 10, 0.0, C.byref(h)) == -1
    for kw in [(0, 1e-4, 10, 0.0), (10, 1e-4, 0, 0.0), (10, 1e-4, 10, -1.0), (10, float("nan"), 10, 0.0)]:
        assert lib().ks_sparse_lbfgs_fit(ctx.handle, sm.handle, y.handle, 1, kw[0], kw[1], kw[2], kw[3], C.byref(h)) == -1, kw
    wrong_d = ks.SparseLinearMapper(np.ones((4, 2)), None, ctx=ctx)
    assert lib().ks_model_apply_sparse(ctx.handle, wrong_d.handle, sm.handle, C.byref(h)) == -1
    with_means = ks.LinearMapper.from_arrays(ctx, np.ones((3, 2)), np.zeros(2), np.zeros(3))
    assert lib().ks_model_apply_sparse(ctx.handle, with_means.handle, sm.handle, C.byref(h)) == -1
    # the dense nodes refuse a SparseMatrix
    with pytest.raises(ks.KeystoneError, match="unsupported dataset type SparseMatrix"):
        ks.BlockLeastSquaresEstimator(2, 1, 0.1, ctx=ctx).fit(sm, y)
    with pytest.raises(ks.KeystoneError, match="unsupported dataset type SparseMatrix"):
        ks.DenseLBFGSwithL2(ctx=ctx).fit(sm, y)
    with pytest.raises(ks.KeystoneError, match="unsupported dataset type SparseMatrix"):
        dense_model.apply(sm)


# ---------------------------------------------------------------------------------------------------------- 7. two ranks
def _worker(rank, world, id_holder, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import keystone_b200 as ks
    rng = np.random.default_rng(8)
    n, d, k = 3001, 4500, 3
    (indptr, indices, data), A = make_sparse(rng, n, d, per_row=30, zipf=True, full_col=True, messy=True, long_rows=3)
    Y = (A[:, :40] @ rng.standard_normal((40, k)) + rng.standard_normal((n, k))).astype(np.float32)

    def rows(r0, r1):
        ip = indptr[r0:r1 + 1] - indptr[r0]
        return (ip, indices[indptr[r0]:indptr[r1]], data[indptr[r0]:indptr[r1]], d), Y[r0:r1]

    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    for name, split in (("uneven", 1000), ("empty", n)):   # rank 1 holds rows [split, n): none in the second fit
        csr, y = rows(0, split) if rank == 0 else rows(split, n)
        est = ks.SparseLBFGSwithL2(num_iterations=8, convergence_tol=0.0, reg_param=0.01, ctx=ctx)
        m = est.fit(ctx.sparse(csr), ctx.matrix(y) if len(y) else ctx.matrix(np.zeros((0, k), np.float32)))
        ret[f"{name}W{rank}"] = np.concatenate(m.xs, 0)
        ret[f"{name}b{rank}"] = m.b_opt
        ret[f"{name}loss{rank}"] = est.loss_history
    ctx.close()
    if rank == 0:
        c1 = ks.Context(device=0)
        e1 = ks.SparseLBFGSwithL2(num_iterations=8, convergence_tol=0.0, reg_param=0.01, ctx=c1)
        m1 = e1.fit(c1.sparse(rows(0, n)[0]), Y)
        ret["W1rank"] = np.concatenate(m1.xs, 0)
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
    for name in ("uneven", "empty"):
        assert np.array_equal(ret[f"{name}W0"], ret[f"{name}W1"]) and np.array_equal(ret[f"{name}b0"], ret[f"{name}b1"])
        assert ret[f"{name}loss0"] == ret[f"{name}loss1"]
        assert _rel(ret[f"{name}W0"], ret["W1rank"]) <= 1e-12
        assert np.allclose(ret[f"{name}loss0"], ret["loss1rank"], rtol=1e-12, atol=0)
