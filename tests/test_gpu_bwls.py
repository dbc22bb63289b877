"""BlockWeightedLeastSquaresEstimator on the device (bwls.cu) against the fp64 oracle (keystone_oracle.bwls_fit) on the
fp32-rounded inputs, at the shapes and class layouts where its own kernels can go wrong: row gather, class ranges that are
not sorted or not aligned, many small classes, b not a multiple of the tile, ragged blocks, several sweeps, the per-class
solves spread over the solve lanes, and the C5 configuration in miniature.

Every case checks W, finalB and the predictions model(F) against F W + finalB, and the fit statistics.  Gates (the library's,
tests/test_gpu_parity.py): parity mode (the default) rel-Frobenius(W) <= 1e-4, "tf32" <= 1.5e-3.  A relative gate on W only
means something when the systems are well conditioned, so every parity case first asserts that an upper bound on the
largest cond(jointXTX_c + lambda I) (bwls_oracle.cond_bound) is <= 1e3.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200._capi import check, lib
from oracle import keystone_oracle as ko

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bwls_oracle as bo  # noqa: E402

pytestmark = pytest.mark.gpu

W_TOL = 1e-4
W_TOL_FAST = 1.5e-3
COND_MAX = 1e3


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------------------------- problems
def zipf_sizes(n, k, rng):
    """Class sizes ~ 1 / rank in a random class order, summing to n, every class present."""
    p = 1.0 / np.arange(1, k + 1)
    s = np.maximum(1, np.floor(n * p / p.sum())).astype(np.int64)
    s[0] += n - s.sum()
    return s[rng.permutation(k)]


def layout(cls, kind, rng):
    """Row order of a class vector: sorted, contiguous runs in a shuffled class order, or interleaved."""
    if kind == "sorted":
        return np.argsort(cls, kind="stable")
    if kind == "runs":
        rank = rng.permutation(cls.max() + 1)
        return np.argsort(rank[cls], kind="stable")
    return rng.permutation(len(cls))


def gaussian_classes(rng, cls, d, k, sep=1.0, offset=0.0):
    """Materialised features: class centroid (sep per coordinate) + unit noise + a common offset, rounded to fp32."""
    cent = sep * rng.standard_normal((k, d))
    return (cent[cls] + rng.standard_normal((len(cls), d)) + offset).astype(np.float32)


def cosine_problem(rng, cls, k, d_in, nrf, n_out, gamma):
    """Inputs with class centroids and `nrf` cosine maps of n_out features; parameters rounded to fp32 as the device keeps them.
    Returns (X32, params, F) with F the fp64 features of the fp32 inputs."""
    X = (0.5 * rng.standard_normal((k, d_in))[cls] + rng.standard_normal((len(cls), d_in))).astype(np.float32)
    params = []
    for _ in range(nrf):
        W, b = ko.cosine_random_features_params(d_in, n_out, gamma, rng)
        params.append((W.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64)))
    F = np.concatenate([ko.cosine_random_features(X.astype(np.float64), W, b) for W, b in params], 1)
    return X, params, F


def generated(ctx, X, params):
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    return ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(ctx.matrix(X))


# ---------------------------------------------------------------------------------------------------------------- checks
def fit_and_check(ctx, data, F, cls, k, bs, iters, lam, w, nf=None, precision="default", tol=W_TOL, cond=True,
                  reshuffled=None, predict=True, ref=None):
    """Fit on the device, compare with the oracle (`ref`: its (xs, finalB) when already computed); returns
    (model, W_device, W_oracle, stats)."""
    Y = ko.class_label_indicators(cls, k)
    if cond and precision == "default":
        cb = bo.cond_bound(F, Y, bs, lam, w, nf)
        assert cb <= COND_MAX, f"systems too ill-conditioned for a relative gate: cond <= {cb:.3g}"
    model = ks.BlockWeightedLeastSquaresEstimator(bs, iters, lam, w, nf, precision=precision).fit(data, ctx.labels_from_classes(cls, k))
    st = ctx.last_fit_stats()
    present = len(np.unique(cls))
    assert st["solver"] == "blockwls" and st["mma"] == ("tf32x2" if precision == "default" else "tf32x1")
    assert st["classes_present"] == present
    assert st["solve_lanes"] == min(present, 4)
    if reshuffled is not None:
        assert st["reshuffled"] == reshuffled
    xs, fb = ref if ref is not None else ko.bwls_fit(F, Y, bs, iters, lam, w, num_features=nf)
    assert [x.shape for x in model.xs] == [x.shape for x in xs]
    assert model.feature_means is None
    Wg, Wr = np.concatenate(model.xs, 0), np.concatenate(xs, 0)
    rel = np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)
    print(f"rel-Fro(W) = {rel:.3e} ({precision}, n={len(cls)}, D={F.shape[1]}, k={k}, b={bs}, iters={iters})")
    assert rel <= tol, rel
    d = Wr.shape[0]
    # finalB = jointLabelMean - sum jointMean W: the W error enters through the feature means
    b_scale = max(1.0, np.abs(fb).max()) + (np.abs(F[:, :d].mean(0)) @ np.abs(Wr)).max()
    assert np.abs(model.b_opt - fb).max() <= tol * b_scale, np.abs(model.b_opt - fb).max()
    if predict:
        pred = model(data).to_numpy()
        ref = F[:, :d] @ Wr + fb
        scale = (np.abs(F[:, :d]) @ np.abs(Wr)).max() + np.abs(fb).max()
        assert np.abs(pred - ref).max() <= tol * scale, np.abs(pred - ref).max() / scale
    return model, Wg, Wr, st


# ---------------------------------------------------------------------------------------------------------------- layouts
@pytest.mark.parametrize("source", ["materialised", "generated"])
@pytest.mark.parametrize("order", ["sorted", "runs", "interleaved"])
def test_class_layouts(ctx, order, source):
    """Class-sorted rows, contiguous runs in a shuffled class order (kept as given: no reshuffle, ranges recomputed) and
    interleaved rows (gathered on the device; generated features: the input rows are gathered and the operands prepared
    again)."""
    rng = np.random.default_rng(11)
    n, k = 6000, 12
    cls = np.sort(rng.choice(k, n, p=np.linspace(2, 1, k) / np.linspace(2, 1, k).sum()))
    X, params, F = cosine_problem(rng, cls, k, 64, 2, 128, 0.25)
    p = layout(cls, order, rng)
    cls, X, F = cls[p], X[p], F[p]
    if source == "materialised":
        F = F.astype(np.float32).astype(np.float64)
        data = ctx.matrix(F.astype(np.float32))
    else:
        data = generated(ctx, X, params)
    fit_and_check(ctx, data, F, cls, k, 128, 2, 1e-2, 0.25, reshuffled=int(order == "interleaved"))


@pytest.mark.parametrize("order", ["sorted", "interleaved"])
def test_rectified_generated_features(ctx, order):
    """MNIST-shaped pipeline: gather(RandomSignNode -> PaddedFFT -> LinearRectifier) x 2 -> VectorCombiner.  Interleaved labels
    gather the input rows into a new generated source, which must keep the rectifier (not fall back to cosines)."""
    rng = np.random.default_rng(5)
    n, d_in, k = 4000, 784, 10
    cls = rng.integers(0, k, n)
    p = layout(cls, order, rng)
    cls = cls[p]
    X = rng.random((n, d_in)).astype(np.float32)
    signs = [2.0 * rng.integers(0, 2, d_in) - 1.0 for _ in range(2)]
    branches = [ks.RandomSignNode(s, ctx).andThen(ks.PaddedFFT(ctx)).andThen(ks.LinearRectifier(0.0, ctx=ctx)) for s in signs]
    feats = ks.Pipeline.gather(branches).andThen(ks.VectorCombiner())(ctx.matrix(X))
    F = ko.mnist_random_fft_features(X.astype(np.float64), signs)
    fit_and_check(ctx, feats, F, cls, k, 512, 1, 10.0, 0.25, reshuffled=int(order == "interleaved"))


# ---------------------------------------------------------------------------------------------------------------- classes
@pytest.mark.parametrize("k,order", [(33, "sorted"), (147, "sorted"), (147, "interleaved")])
def test_class_sizes(ctx, k, order):
    """Zipf-like class sizes with a 1-row class, a 31-row class and empty classes between present ones; class ranges start at
    rows that are not multiples of 32; kpad > 32 and more classes than solve lanes."""
    rng = np.random.default_rng(k)
    sizes = zipf_sizes(5000, k, rng)
    sizes[[3, 8, k - 2]] = 0
    sizes[5], sizes[9] = 1, 31
    cls = np.repeat(np.arange(k), sizes)
    cls = cls[layout(cls, order, rng)]
    F = gaussian_classes(rng, cls, 96, k).astype(np.float64)
    starts = np.r_[0, np.cumsum(sizes[sizes > 0])[:-1]]
    assert (starts % 32 != 0).sum() > len(starts) // 2
    model, Wg, _, _ = fit_and_check(ctx, ctx.matrix(F.astype(np.float32)), F, cls, k, 64, 2, 0.05, 0.25,
                                    reshuffled=int(order == "interleaved"))
    assert np.all(Wg[:, sizes == 0] == 0.0)          # classes without rows keep W = 0


# ---------------------------------------------------------------------------------------------------------------- blocks
@pytest.mark.parametrize("bs,D,nf,iters,w", [
    (200, 450, None, 1, 0.25),     # b % 32 != 0, two 128-wide tiles, ragged last block (50)
    (200, 600, 450, 3, 0.75),      # num_features_opt < D, ragged, three sweeps
    (512, 1100, None, 3, 0.75),    # ragged last block (76)
    (512, 512, None, 1, 0.25),
])
def test_blocks(ctx, bs, D, nf, iters, w):
    rng = np.random.default_rng(bs + D)
    n, k = 3000, 8
    cls = rng.integers(0, k, n)
    F = gaussian_classes(rng, cls, D, k, sep=0.5).astype(np.float64)
    fit_and_check(ctx, ctx.matrix(F.astype(np.float32)), F, cls, k, bs, iters, 0.05, w, nf=nf, reshuffled=1)


# ---------------------------------------------------------------------------------------------------------------- lanes
def test_solve_lanes_agree(ctx):
    """The per-class solves on 1, 4 (default) and 16 lanes: each matches the oracle, and all agree to 1e-6 (not bit-equal: the
    order of the Gram's reduction varies between runs)."""
    rng = np.random.default_rng(21)
    n, k = 4000, 33
    cls = np.sort(rng.integers(0, k, n))
    F = gaussian_classes(rng, cls, 128, k).astype(np.float64)
    data = ctx.matrix(F.astype(np.float32))
    Ws = {}
    try:
        for lanes in (1, 16, 4):
            ctx.set_option("solve_lanes", lanes)
            model = ks.BlockWeightedLeastSquaresEstimator(128, 2, 0.05, 0.25).fit(data, ctx.labels_from_classes(cls, k))
            assert ctx.last_fit_stats()["solve_lanes"] == lanes
            Ws[lanes] = np.concatenate(model.xs, 0)
    finally:
        ctx.set_option("solve_lanes", 4)
    xs, _ = ko.bwls_fit(F, ko.class_label_indicators(cls, k), 128, 2, 0.05, 0.25)
    Wr = np.concatenate(xs, 0)
    for lanes, Wg in Ws.items():
        assert np.linalg.norm(Wg - Wr) <= W_TOL * np.linalg.norm(Wr), lanes
        assert np.linalg.norm(Wg - Ws[4]) <= 1e-6 * np.linalg.norm(Ws[4]), lanes


# ---------------------------------------------------------------------------------------------------------------- C5
C5 = dict(n=64000, d_in=440, nrf=2, n_out=1024, k=147, lam=6e-5, w=0.25, bs=1024)


@pytest.fixture(scope="module")
def c5_problem():
    """Config 5 in miniature: class-sorted rows with Zipf class sizes, 2 x 1024 cosine features of 440 inputs, k = 147,
    lambda = 6e-5 and w = 0.25 (the reference's ImageNet defaults), b = 1024."""
    rng = np.random.default_rng(147)
    sizes = zipf_sizes(C5["n"], C5["k"], rng)
    cls = np.repeat(np.arange(C5["k"]), sizes)
    X, params, F = cosine_problem(rng, cls, C5["k"], C5["d_in"], C5["nrf"], C5["n_out"], 0.1)
    ref = ko.bwls_fit(F, ko.class_label_indicators(cls, C5["k"]), C5["bs"], 1, C5["lam"], C5["w"])
    return cls, X, params, F, ref


@pytest.mark.parametrize("precision,tol", [("default", W_TOL), ("tf32", W_TOL_FAST)])
def test_c5_miniature(ctx, c5_problem, precision, tol):
    cls, X, params, F, ref = c5_problem
    fit_and_check(ctx, generated(ctx, X, params), F, cls, C5["k"], C5["bs"], 1, C5["lam"], C5["w"], precision=precision, tol=tol,
                  reshuffled=0, ref=ref)


def test_f16_precision_is_the_tf32_mode(ctx):
    """precision="f16" is accepted by the weighted solver and computes as "tf32" does (one tf32 MMA per product): bit-equal on
    materialised features.  On generated features the shift is a sampled mean summed with fp32 atomics, so its last bits, and
    with them the tf32 rounding of the slab, vary between runs (two "tf32" fits differ by 7e-5 on an H100): there the two modes
    must agree within that spread, far below the fast-mode gate."""
    rng = np.random.default_rng(16)
    n, k = 3000, 6
    cls = rng.integers(0, k, n)
    X, params, F = cosine_problem(rng, cls, k, 32, 1, 160, 0.25)
    for source in ("materialised", "generated"):
        if source == "materialised":
            Fs = F.astype(np.float32).astype(np.float64)
            data = ctx.matrix(F.astype(np.float32))
        else:
            Fs, data = F, generated(ctx, X, params)
        Wm = {}
        for prec in ("tf32", "f16"):
            _, Wm[prec], _, _ = fit_and_check(ctx, data, Fs, cls, k, 96, 2, 1e-2, 0.25, precision=prec, tol=W_TOL_FAST)
        if source == "materialised":
            assert np.array_equal(Wm["f16"], Wm["tf32"])
        else:
            assert np.linalg.norm(Wm["f16"] - Wm["tf32"]) <= W_TOL_FAST / 5 * np.linalg.norm(Wm["tf32"])


# ---------------------------------------------------------------------------------------------------------------- errors
def test_not_positive_definite_raises_and_context_recovers(ctx):
    """lambda = 0 and w = 1: the system of a 1-row class is its (zero) covariance.  The fit must fail with KS_ERR_NOT_SPD and the
    same context must then fit the next problem correctly."""
    rng = np.random.default_rng(7)
    cls = np.r_[np.zeros(200, np.int64), np.ones(1, np.int64), np.full(150, 2)]
    F = gaussian_classes(rng, cls, 40, 3)
    with pytest.raises(ks.KeystoneError) as e:
        ks.BlockWeightedLeastSquaresEstimator(20, 1, 0.0, 1.0).fit(ctx.matrix(F), ctx.labels_from_classes(cls, 3))
    assert e.value.code == -7
    cls2 = rng.integers(0, 5, 2000)
    F2 = gaussian_classes(rng, cls2, 70, 5).astype(np.float64)
    fit_and_check(ctx, ctx.matrix(F2.astype(np.float32)), F2, cls2, 5, 32, 2, 0.05, 0.3, reshuffled=1)


# ---------------------------------------------------------------------------------------------------------------- separated classes
@pytest.fixture(scope="module")
def separated_problem():
    """Class centroids 1.5 within-class sigma apart per coordinate and a common column offset of 50: after the shift by the
    population mean, every row of a class carries its centroid offset, so the class Grams and S_c^T r_c are sums of same-sign
    products -- where the tensor core's truncating fp32 accumulation is biased."""
    rng = np.random.default_rng(50)
    k = 20
    sizes = zipf_sizes(50000, k, rng)
    cls = np.repeat(np.arange(k), sizes)
    F = gaussian_classes(rng, cls, 256, k, sep=1.5, offset=50.0)
    return cls, F


@pytest.mark.xfail(strict=True, reason="rel-Fro(W) = 7.5e-4 > 1e-4 on an H100: with the diagonals exact (captured |dH_ii| 8e-12), "
                   "the off-diagonal class-Gram entries and S_c^T r_c still carry the truncation bias of the class-mean offsets "
                   "(~0.3 of the system_bounds bound); removing the class mean before the tensor core is the open fix")
def test_separated_classes(ctx, separated_problem):
    cls, F32 = separated_problem
    F = F32.astype(np.float64)
    fit_and_check(ctx, ctx.matrix(F32), F, cls, 20, 256, 2, 1e-2, 0.25, reshuffled=0)


# ---------------------------------------------------------------------------------------------------------------- capture
CHUNK = 2048   # rows per accumulation chain of the parity mode's class Grams (bwls.cu)


def capture(ctx, data, cls, k, bs, lam, w, block, c, b):
    H = np.full((b, b), np.nan, order="F")
    r = np.full(b, np.nan)
    check(ctx.handle, lib().ks_debug_bwls_capture(ctx.handle, block, c, H.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p)))
    ks.BlockWeightedLeastSquaresEstimator(bs, 1, lam, w).fit(data, ctx.labels_from_classes(cls, k))
    assert not np.isnan(H).any() and not np.isnan(r).any(), "nothing captured"
    return np.array(H), r


def system_bounds(F, cls, k, bs, w, block, c):
    """Entrywise bounds on |H_device - H| and |rhs_device - rhs| for class c of feature block `block` at the first sweep.

    The device shifts the block by m (here the population mean, as for materialised features) and forms S = fl32(F - m), one
    fp32 rounding: <= 2^-24 |S|.  S and the residual R (fp32 of labels - jointLabelMean) are carried as tf32 pairs hi + lo,
    which represent them to 2^-22 relative; the MMA keeps hi*hi + hi*lo + lo*hi and drops lo*lo (<= 2^-22 |a||b|).  The
    tensor core adds each 8-deep product group into the fp32 accumulator with at most one ulp of error, 2^-23 of the partial
    sum, which is bounded by the sum of |products|; a chain is CHUNK rows long, so CHUNK / 8 additions.  The chains and the
    classes are then summed and stored in fp32: one 2^-24 rounding per addition, (rows / CHUNK + k + 1) of them.  So for an
    entry of a Gram over `n` rows
        |G_dev - G| <= eps(n) * (|S|^T |S|)_rc,   eps(n) = 2^-23 + 3 * 2^-22 + (CHUNK / 8) * 2^-23 + (n / CHUNK + k + 1) * 2^-24
    and the same for S^T R with |S|^T |R|.  The fp64 assembly (H = (1-w)(Gpop/N - dp dp^T) + w(Gc/nc - dc dc^T) + ...)
    divides the Gram bounds by N and nc; the means dp, dc are fp64 sums of the same pairs (2^-21 relative, a term far below
    the rest), and the raw-feature correction m * sum(r) adds 2^-23 |m| sum|r| from the fp32 residual."""
    Y = ko.class_label_indicators(cls, k)
    n = len(cls)
    counts = np.bincount(cls, minlength=k)
    jlm = np.where(counts > 0, 2 * w + 2 * (1.0 - w) * counts / n - 1, 0.0)
    R = Y - jlm
    s0, e0 = ko.block_bounds(F.shape[1], bs)[block]
    A = F[:, s0:e0]
    m = A.mean(axis=0).astype(np.float32).astype(np.float64)
    S = np.abs(A - m)
    sel = cls == c
    nc = sel.sum()

    def eps(rows):
        return 2.0 ** -23 + 3 * 2.0 ** -22 + (CHUNK / 8) * 2.0 ** -23 + (rows / CHUNK + k + 1) * 2.0 ** -24

    Sc = S[sel]
    absR = np.abs(R)
    dp, dc = S.mean(0), Sc.mean(0)
    small = 2.0 ** -20 * ((1 - w) * np.outer(dp, dp) + w * np.outer(dc, dc) + w * (1 - w) * np.outer(dc + dp, dc + dp))
    bH = (1 - w) * eps(n) * (S.T @ S) / n + w * eps(nc) * (Sc.T @ Sc) / nc + small
    bR = ((1 - w) * eps(n) * (S.T @ absR[:, c]) / n + w * eps(nc) * (Sc.T @ absR[sel, c]) / nc
          + 2.0 ** -23 * np.abs(m) * ((1 - w) * absR[:, c].mean() + w * absR[sel, c].mean()))
    return bH, bR


def check_capture(ctx, F32, cls, k, bs, lam, w):
    F = F32.astype(np.float64)
    data = ctx.matrix(F32)
    counts = np.bincount(cls, minlength=k)
    c_small = int(np.argmin(np.where(counts > 0, counts, counts.max() + 1)))
    c_big = int(np.argmax(counts))
    nb = len(ko.block_bounds(F.shape[1], bs))
    for block, c in [(0, c_small), (0, c_big), (nb - 1, c_small)]:
        b = ko.block_bounds(F.shape[1], bs)[block][1] - ko.block_bounds(F.shape[1], bs)[block][0]
        H, r = capture(ctx, data, cls, k, bs, lam, w, block, c, b)
        Href, rref = bo.reference_systems(F, ko.class_label_indicators(cls, k), bs, lam, w, block, classes=[c])[c]
        bH, bR = system_bounds(F, cls, k, bs, w, block, c)
        errH = np.abs(H - Href)
        dg = np.diag(errH) / np.diag(bH)
        off = (errH / bH)[~np.eye(b, dtype=bool)]
        print(f"capture block {block} class {c} (n_c = {counts[c]}): |dH| diag max {np.diag(errH).max():.3e} "
              f"({dg.max():.3f} of bound), off-diag {off.max():.3f} of bound; bound diag max {np.diag(bH).max():.3e}")
        assert (errH <= bH).all(), (dg.max(), off.max())
        # the bound is far below the terms the device must get right, so dropping any of them fails
        s0, e0 = ko.block_bounds(F.shape[1], bs)[block]
        A = F[:, s0:e0]
        f = A[cls == c]
        cov_diag = w * ((f - f.mean(0)) ** 2).mean(0)
        md = f.mean(0) - A.mean(0)
        mix_term = w * (1 - w) * np.outer(md, md)
        assert bH.max() < 1e-2 * cov_diag.min(), (bH.max(), cov_diag.min())
        assert bH.max() < 1e-2 * np.abs(mix_term).max(), (bH.max(), np.abs(mix_term).max())
        assert (np.abs(np.diag(H) - (np.diag(Href) - cov_diag)) > np.diag(bH)).all()
        assert (np.abs(H - (Href - mix_term)) > bH).any()
        if block == 0:
            errR = np.abs(r - rref)
            print(f"  |drhs| max {errR.max():.3e} ({(errR / bR).max():.3f} of bound)")
            assert (errR <= bR).all(), (errR / bR).max()
            assert bR.max() < 1e-2 * np.abs(rref).max()


def test_capture_separated_classes(ctx, separated_problem):
    """The assembled fp64 system of a small and of the largest class against jointXTX + lambda I and jointXTR of the oracle,
    entrywise within the bound derived from the operand format and the chain length (system_bounds)."""
    cls, F32 = separated_problem
    check_capture(ctx, F32, cls, 20, 256, 1e-2, 0.25)


def test_capture_c5_miniature(ctx, c5_problem):
    """The same on the C5 miniature's features, materialised in fp32 (the bound is stated for a known slab)."""
    cls, _, _, F, _ = c5_problem
    check_capture(ctx, F.astype(np.float32), cls, C5["k"], C5["bs"], C5["lam"], C5["w"])
