"""PCA, ZCA whitening and approximate PCA on the H100 through the C ABI / node API, against the fp64 oracle (tests/pca_oracle.py) on
the same fp32 inputs.  The fits run in fp64 on the DMMA tensor core, so the gates are fp64-sized: the Gram to 1e-12 max|G|, pca_mat
to 1e-8, eigenvalues to 1e-10 relative, the whitener to 1e-8 relative (Frobenius)."""
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
import pca_oracle as po  # noqa: E402


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


def _gram_f64(ctx, A, B=None, sa=None, sb=None):
    from keystone_b200._capi import lib, check
    a = ctx.matrix(A.astype(np.float32))
    b = ctx.matrix(B.astype(np.float32)) if B is not None else None
    m, n = A.shape[1], (B if B is not None else A).shape[1]
    out = np.empty((m, n))
    sa = None if sa is None else np.ascontiguousarray(sa, dtype=np.float64)
    sb = None if sb is None else np.ascontiguousarray(sb, dtype=np.float64)
    pa = None if sa is None else sa.ctypes.data_as(C.c_void_p)
    pb = None if sb is None else sb.ctypes.data_as(C.c_void_p)
    check(ctx.handle, lib().ks_debug_gram_f64(ctx.handle, a.handle, 0 if b is None else b.handle, pa, pb,
                                              out.ctypes.data_as(C.c_void_p), n))
    return out


# ---------------------------------------------------------------------------------------------------------- 1. the DMMA Gram
@pytest.mark.parametrize("N", [1, 31, 4097, 100003])
@pytest.mark.parametrize("m", [1, 10, 108, 130, 257])
def test_gram_f64_matches_numpy(ctx, N, m):
    rng = np.random.default_rng(N * 1000 + m)
    A = _f32(rng.standard_normal((N, m)) + 2.0)
    s = A.mean(0)
    for sa in (None, s):
        G = _gram_f64(ctx, A, None, sa)
        Ac = A - (0 if sa is None else sa)
        ref = Ac.T @ Ac
        assert np.array_equal(G, G.T)
        assert np.abs(G - ref).max() <= 1e-12 * np.abs(ref).max(), (sa is None, np.abs(G - ref).max() / np.abs(ref).max())
    for n in (1, 25):
        B = _f32(rng.standard_normal((N, n)) - 1.0)
        t = B.mean(0)
        for sa, sb in ((None, None), (s, t)):
            G = _gram_f64(ctx, A, B, sa, sb)
            ref = (A - (0 if sa is None else sa)).T @ (B - (0 if sb is None else sb))
            assert np.abs(G - ref).max() <= 1e-12 * np.abs(ref).max()


# ---------------------------------------------------------------------------------------------------------- 2. transformers
def test_pca_transformer_known_answer(ctx):
    """PCASuite "PCA matrix transformation" (T/nodes/learning/PCASuite.scala:15-50): exact integers."""
    import keystone_b200 as ks
    pca = ks.PCATransformer.from_matrix(ctx, np.array([[1, 2], [3, 4], [5, 6], [7, 8]], dtype=np.float64))
    one = np.arange(12, dtype=np.float64).reshape(4, 3).T          # Breeze column-major 3 x 4 of 0 .. 11
    two = np.ones((8, 4))
    out = pca.apply(np.concatenate([one, two]).astype(np.float32)).to_numpy()
    assert np.array_equal(out[:3], [[102, 120], [118, 140], [134, 160]])
    assert np.array_equal(out[3:], np.tile([16.0, 20.0], (8, 1)))
    batch = ks.BatchPCATransformer(pca)
    rng = np.random.default_rng(1)
    items = [rng.integers(-5, 5, (4, m)).astype(np.float64) for m in (1, 7, 3)]
    res = batch.apply(items)
    assert [r.shape for r in res] == [(2, 1), (2, 7), (2, 3)]
    for it, r in zip(items, res):
        assert np.array_equal(r, pca.pca_mat.T @ it)


# ---------------------------------------------------------------------------------------------------------- 3. exact PCA
@pytest.mark.parametrize("n,d,dims", [(1000, 10, 5), (100003, 130, 80), (20000, 1000, 100)])
def test_pca_matches_oracle(ctx, n, d, dims):
    import keystone_b200 as ks
    X = po.planted(n, d, dims, np.random.default_rng(n + d))
    est = ks.PCAEstimator(dims, ctx=ctx)
    m = est.fit(X.astype(np.float32))
    P = m.pca_mat
    ref = po.compute_pca(X, dims)
    assert P.shape == (d, dims) and m.b_opt is None and m.feature_means is None
    assert np.abs(P - ref).max() <= 1e-8, np.abs(P - ref).max()
    lam = po.singular_values_sq(X)[:dims]
    assert np.abs(est.eigenvalues - lam).max() <= 1e-10 * lam.max()
    st = ctx.last_fit_stats()
    for key in ("mean_ms", "gram_ms", "allreduce_ms", "eig_ms", "qr_ms", "n_total", "d", "dims", "l", "q", "eigenvalues"):
        assert key in st, key
    assert st["n_total"] == n and st["d"] == d and st["dims"] == dims
    if d <= 130:   # PCASuite "PCA Estimation": the reduced data has a diagonal covariance
        assert po.off_diagonal_cov(m.apply(X.astype(np.float32)).to_numpy()) < 1e-4 * max(1.0, lam[0] / n)


def test_suite_pca_estimation(ctx):
    """PCASuite "PCA Estimation" and "Covariance Matrix of Distributed PCA should match local one" (1000 x 10 -> 5)."""
    import keystone_b200 as ks
    X = _f32(np.random.default_rng(2).standard_normal((1000, 10)))
    local = ks.PCAEstimator(5, ctx=ctx).fit(X.astype(np.float32))
    dist = ks.DistributedPCAEstimator(5, ctx=ctx).fit(X.astype(np.float32))
    assert po.off_diagonal_cov(local.apply(X.astype(np.float32)).to_numpy()) < 1e-4
    assert np.abs(local.pca_mat - dist.pca_mat).max() < 1e-4
    assert np.abs(local.pca_mat - po.distributed_pca(np.array_split(X, 4), 5)).max() < 1e-8


# ---------------------------------------------------------------------------------------------------------- 4. ZCA
def _patches(rng, n_img, conv=6):
    """Row-normalised 6 x 6 x 3 patches of random images (Stats.normalizeRows(., 10)): every row sums to zero, so the covariance is
    rank-deficient."""
    from oracle import keystone_oracle as ko
    imgs = rng.integers(0, 256, (n_img, 32, 32, 3)).astype(np.float64)
    pts = np.concatenate([ko.make_patches(im, conv, normalize=False) for im in imgs], 0)
    return pts, imgs


def test_zca_matches_oracle(ctx):
    import keystone_b200 as ks
    from oracle import keystone_oracle as ko
    rng = np.random.default_rng(3)
    X = po.planted(20000, 108, 30, rng)
    for data, eps in ((X, 0.1), (None, 1e-5)):
        if data is None:
            pts, _ = _patches(rng, 8)
            data = _f32(ko.normalize_rows(pts[rng.choice(pts.shape[0], 5000, replace=False)], 10.0))
            assert np.abs(data.sum(1)).max() < 1e-4      # the null direction the tensor-core Gram would lose
        est = ks.ZCAWhitenerEstimator(eps, ctx=ctx)
        w = est.fit_single(data.astype(np.float32))
        Wr, mr = po.zca_fit(data, eps)
        assert _rel(w.whitener, Wr) <= 1e-8, _rel(w.whitener, Wr)
        assert np.abs(w.means - mr).max() <= 1e-12 * np.abs(mr).max()
        assert w.b_opt is None
        got = w.apply(data.astype(np.float32)).to_numpy()       # (x - means) * whitener in the context's precision
        ref = po.zca_apply(data, Wr, mr)
        assert _rel(got, ref) <= 1e-5


def test_suite_zca_eps(ctx):
    """ZCAWhiteningSuite (T/nodes/learning/ZCAWhiteningSuite.scala): 10 000 x 10 Gaussian."""
    import keystone_b200 as ks
    X = _f32(np.random.default_rng(4).standard_normal((10000, 10)))

    def dev(eps):
        w = ks.ZCAWhitenerEstimator(eps, ctx=ctx).fit_single(X.astype(np.float32))
        return np.abs(np.cov(po.zca_apply(X, w.whitener, w.means), rowvar=False) - np.eye(10)).max()

    assert dev(1e-12) < 1e-4
    assert dev(0.1) < 0.1 and not dev(0.1) < 1e-4


# ---------------------------------------------------------------------------------------------------------- 5. CIFAR front end
def test_random_patch_cifar_front_end(ctx):
    """RandomPatchCifar.scala:45-63 in miniature: sampled patches -> normalizeRows -> ZCA fit (device) -> whitened, normalised
    filters times whitener^T -> Convolver(filters, whitener.means) -> SymmetricRectifier -> Pooler, vs the oracle's whole chain."""
    import keystone_b200 as ks
    from oracle import keystone_oracle as ko
    rng = np.random.default_rng(6)
    pts, imgs = _patches(rng, 24)
    base = _f32(ko.normalize_rows(pts[rng.choice(pts.shape[0], 4000, replace=False)], 10.0))
    eps, nf = 1e-5, 64
    w = ks.ZCAWhitenerEstimator(eps, ctx=ctx).fit_single(base.astype(np.float32))
    sample = base[rng.choice(base.shape[0], nf, replace=False)]

    def filters_of(unnorm, whitener):
        return (unnorm / (np.sqrt((unnorm ** 2).sum(1)) + 1e-10)[:, None]) @ whitener.T

    # the pipeline whitens its 64-row filter sample on the driver (a local DenseMatrix): on the host here too, with the device's
    # whitener.  (The device apply runs in the context's precision, whose ~2^-21 operand error the eps = 1e-5 null direction
    # amplifies to ~1e-3 of these filters.)
    filt = filters_of(po.zca_apply(sample, w.whitener, w.means), w.whitener)
    Wr, mr = po.zca_fit(base, eps)
    filt_ref = filters_of(po.zca_apply(sample, Wr, mr), Wr)
    assert _rel(filt, filt_ref) <= 1e-6, _rel(filt, filt_ref)
    conv = ks.Convolver(ctx, filt, 32, 32, 3, w.means, normalize_patches=True, var_constant=10.0)
    chain = conv.andThen(ks.SymmetricRectifier(alpha=0.25)).andThen(ks.Pooler(13, 14)).andThen(ks.ImageVectorizer())
    got = chain(ctx.matrix(ks.images_to_matrix(imgs[:8]))).to_numpy()
    ref = np.stack([ko.random_patch_cifar_features(im, filt_ref, mr, 6, 0.25, 13, 14) for im in imgs[:8]])
    assert np.abs(got - ref).max() < 1e-4 * np.abs(ref).max(), np.abs(got - ref).max() / np.abs(ref).max()


# ---------------------------------------------------------------------------------------------------------- 6. approximate PCA
def test_approximate_pca_matches_oracle(ctx):
    import keystone_b200 as ks
    n, d, dims, q, p = 5000, 300, 10, 4, 5
    X = po.planted(n, d, dims, np.random.default_rng(7), mean_scale=0.0)
    est = ks.ApproximatePCAEstimator(dims, q=q, p=p, seed=11, ctx=ctx)
    P = est.fit(X.astype(np.float32)).pca_mat
    om = po.omega(d, dims + p, 11)
    ref = po.approximate_pca(X, om, dims, q)
    assert np.abs(P - ref).max() <= 1e-8, np.abs(P - ref).max()
    st = ctx.last_fit_stats()
    assert st["l"] == dims + p and st["q"] == q and len(st["singular_values"]) == dims
    # approximateQ: orthonormal (fp32 output) and the oracle's projector
    Q = ks.ApproximatePCAEstimator.approximate_q(X.astype(np.float32), dims + p, q, seed=11, ctx=ctx).to_numpy()
    Qr = po.approximate_q(X, om, q)
    assert np.abs(Q.T @ Q - np.eye(dims + p)).max() <= 1e-6
    assert np.abs(Q @ Q.T - Qr @ Qr.T).max() <= 1e-6


def test_approximate_q_exactly_low_rank(ctx):
    """l = 15 > rank 3: the sketch is exactly rank-deficient; shifted CholeskyQR3 does not fail and still spans the data."""
    import keystone_b200 as ks
    rng = np.random.default_rng(8)
    X = _f32(rng.standard_normal((400, 3)) @ rng.standard_normal((3, 60)))
    Q = ks.ApproximatePCAEstimator.approximate_q(X.astype(np.float32), 15, 2, seed=1, ctx=ctx).to_numpy()
    assert np.isfinite(Q).all()
    assert np.abs(Q.T @ Q - np.eye(15)).max() <= 1e-5
    assert np.linalg.norm(X - Q @ (Q.T @ X)) <= 1e-5 * np.linalg.norm(X)
    assert ctx.last_fit_stats()["shifted_qr_passes"] >= 3
    P = ks.ApproximatePCAEstimator(3, q=2, p=12, seed=1, ctx=ctx).fit(X.astype(np.float32)).pca_mat
    assert np.isfinite(P).all() and np.abs(P.T @ P - np.eye(3)).max() <= 1e-8


def test_suite_approximate_assertions(ctx):
    """PCASuite: the HMT sketch bound over a (p, k, q) grid, singular values within mre 0.05 of the exact PCA's, and an approximate
    off-diagonal covariance below 0.1 (200 x 100 Gaussian, dims 10)."""
    import keystone_b200 as ks
    X = _f32(np.random.default_rng(9).standard_normal((200, 100)))
    s = np.linalg.svd(X, compute_uv=False)
    for p in (5, 10):
        for k in (1, 5, 10, 20):
            for q in (1, 5, 20):
                Q = ks.ApproximatePCAEstimator.approximate_q(X.astype(np.float32), k + p, q, seed=p + k + q, ctx=ctx).to_numpy()
                Q = Q.astype(np.float64)
                assert np.linalg.norm(X - Q @ (Q.T @ X)) < (1 + 9 * np.sqrt(k + p) * 100) * s[k]
    approx = ks.ApproximatePCAEstimator(10, q=10, ctx=ctx).fit(X.astype(np.float32)).apply(X.astype(np.float32)).to_numpy()
    exact = ks.PCAEstimator(10, ctx=ctx).fit(X.astype(np.float32)).apply(X.astype(np.float32)).to_numpy()
    sa, se = np.linalg.svd(approx, compute_uv=False), np.linalg.svd(exact, compute_uv=False)
    assert np.mean(np.abs(sa - se) / np.abs(se)) < 0.05
    assert po.off_diagonal_cov(approx) < 0.1


# ---------------------------------------------------------------------------------------------------------- 7. model plumbing
def test_model_plumbing(ctx, tmp_path):
    import keystone_b200 as ks
    X = po.planted(3000, 64, 8, np.random.default_rng(10))
    m = ks.PCAEstimator(8, ctx=ctx).fit(X.astype(np.float32))
    P = m.pca_mat
    assert _rel(m.apply(X.astype(np.float32)).to_numpy(), X @ P) <= 1e-5
    ctx.set_option("precision", 1)
    try:
        assert _rel(m.apply(X.astype(np.float32)).to_numpy(), X @ P) <= 1.5e-3
    finally:
        ctx.set_option("precision", 2)
    w = ks.ZCAWhitenerEstimator(0.1, ctx=ctx).fit(X.astype(np.float32))
    assert _rel(w.apply(X.astype(np.float32)).to_numpy(), (X - w.means) @ w.whitener) <= 1e-5
    for model, cls in ((m, ks.PCATransformer), (w, ks.ZCAWhitener)):
        path = str(tmp_path / f"{cls.__name__}.ksm")
        model.save(path)
        back = cls.load(ctx, path)
        assert np.array_equal(back.x, model.x)
        assert (back.feature_means is None) == (model.feature_means is None)
    assert np.array_equal(ks.ZCAWhitener.load(ctx, str(tmp_path / "ZCAWhitener.ksm")).means, w.means)
    st = ctx.last_fit_stats()
    assert st["solver"] == "zca" and len(st["eigenvalues"]) == 64


# ---------------------------------------------------------------------------------------------------------- 8. rejections
def test_rejections(ctx):
    import keystone_b200 as ks
    from keystone_b200._capi import lib
    x = ctx.matrix(np.random.default_rng(0).standard_normal((20, 6)).astype(np.float32))
    small = ctx.matrix(np.ones((5, 6), dtype=np.float32))
    om = np.asfortranarray(np.ones((6, 8)))
    op = om.ctypes.data_as(C.c_void_p)
    h = C.c_int64(0)
    assert lib().ks_pca_fit(ctx.handle, x.handle, 3, C.byref(h)) == 0
    ks.PCATransformer(ctx, h.value)
    for dims in (0, -1, 7):
        assert lib().ks_pca_fit(ctx.handle, x.handle, dims, C.byref(h)) == -1
    assert lib().ks_zca_fit(ctx.handle, small.handle, 0.1, C.byref(h)) == -1          # N < d
    for eps in (-1e-3, float("nan"), float("inf")):
        assert lib().ks_zca_fit(ctx.handle, x.handle, eps, C.byref(h)) == -1
    assert lib().ks_approx_range(ctx.handle, x.handle, op, 7, 1, C.byref(h)) == -1      # l > d
    assert lib().ks_approx_range(ctx.handle, small.handle, op, 6, 1, C.byref(h)) == -1  # l > N
    assert lib().ks_approx_range(ctx.handle, x.handle, op, 4, -1, C.byref(h)) == -1     # q < 0
    assert lib().ks_approx_range(ctx.handle, x.handle, None, 4, 1, C.byref(h)) == -1    # null omega
    assert lib().ks_approx_pca_fit(ctx.handle, x.handle, op, 0, 1, 2, C.byref(h)) == -1
    assert lib().ks_approx_pca_fit(ctx.handle, x.handle, op, 3, 1, 4, C.byref(h)) == -1  # l = 7 > d
    assert lib().ks_approx_pca_fit(ctx.handle, x.handle, None, 3, 1, 2, C.byref(h)) == -1
    rf = ks.CosineRandomFeatures(ctx, np.ones((4, 6)), np.zeros(4))                   # a feature-map handle is not a matrix
    assert lib().ks_pca_fit(ctx.handle, rf.handle, 2, C.byref(h)) == -6
    assert lib().ks_zca_fit(ctx.handle, 987654, 0.1, C.byref(h)) == -6
    with pytest.raises(ValueError):
        ks.ZCAWhitenerEstimator(-1.0)
    with pytest.raises(ValueError):
        ks.ApproximatePCAEstimator(3, q=-1)
    with pytest.raises(ks.KeystoneError):
        ks.PCAEstimator(9, ctx=ctx).fit(x)


# ---------------------------------------------------------------------------------------------------------- 9. two ranks
def _worker(rank, world, id_holder, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import keystone_b200 as ks
    import pca_oracle as po2
    X = po2.planted(3001, 130, 20, np.random.default_rng(12)).astype(np.float32)
    rows = np.r_[0:100] if rank == 0 else np.r_[100:3001]     # rank 0 holds fewer rows than d
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    ret[f"pca{rank}"] = ks.PCAEstimator(20, ctx=ctx).fit(X[rows]).pca_mat.copy()
    w = ks.ZCAWhitenerEstimator(0.1, ctx=ctx).fit_single(X[rows])
    ret[f"zca{rank}"] = (w.whitener.copy(), w.means.copy())
    ret[f"apx{rank}"] = ks.ApproximatePCAEstimator(20, q=3, p=5, ctx=ctx).fit(X[rows]).pca_mat.copy()
    ctx.close()
    if rank == 0:
        c1 = ks.Context(device=0)
        ret["pca1r"] = ks.PCAEstimator(20, ctx=c1).fit(X).pca_mat.copy()
        w1 = ks.ZCAWhitenerEstimator(0.1, ctx=c1).fit_single(X)
        ret["zca1r"] = (w1.whitener.copy(), w1.means.copy())
        ret["apx1r"] = ks.ApproximatePCAEstimator(20, q=3, p=5, ctx=c1).fit(X).pca_mat.copy()
        c1.close()


def test_two_rank_fits_equal_one_rank():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import keystone_b200 as ks
    mgr = mp.Manager()
    id_holder = mgr.dict(); ret = mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    for key in ("pca", "apx"):
        assert np.array_equal(ret[f"{key}0"], ret[f"{key}1"])
        assert _rel(ret[f"{key}0"], ret[f"{key}1r"]) <= 1e-12
    (w0, m0), (w1, m1), (wr, mr) = ret["zca0"], ret["zca1"], ret["zca1r"]
    assert np.array_equal(w0, w1) and np.array_equal(m0, m1)
    assert _rel(w0, wr) <= 1e-12 and _rel(m0, mr) <= 1e-12
