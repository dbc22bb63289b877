"""fp64 restatement of the block least-squares fit's step algebra (engine.cu::fit_blockls) and the entrywise error bounds of
each step, shared by tests/test_gpu_blockls_steps.py (against states captured from a device fit, ks_debug_blockls_capture) and
tests/test_blockls_steps_algebra.py (the same functions rehearsed on the CPU).

Per block j the device shifts the features by m_j (generated features: the mean of the first `sample_rows` rows of every rank;
materialised features: the exact column mean) and stores the slab as one or two planes, S_hat = hi + lo.  With
delta = mean(S_hat) (from fp32 column sums), N the row count and R the fp32 residual before the step:
    H   = S_hat^T S_hat - N delta delta^T + lambda I                       (sweep 0; later sweeps reuse the factor)
    rhs = S_hat^T R - delta rsum^T - lambda W_old,  rsum = 1^T R           (= (S_hat - 1 delta^T)^T R - lambda W_old)
    dW  = H^-1 rhs,  W_j += dW
    R  -= S_hat dW - 1 cbias^T,  cbias = delta^T dW                         (= R - (S_hat - 1 delta^T) dW)
    mean_j = m_j + delta
The bounds count the device's arithmetic: the dropped lo * lo product, the operand split of R and dW (10-bit in the fast modes,
~21-bit pairs in the parity mode, with the fp16 modes' power-of-two scales and subnormal lo), one fp32 ulp per 8-deep
tensor-core accumulation group along a chain of `chain` rows (or of the block width in the update), the fp32 reduce-adds of the
chains and the fp32 column sums and atomics.
"""
import numpy as np

EPS32 = 2.0 ** -24
EPS64 = 2.0 ** -53

# operand modes of the fit (the "mma" field of its statistics): (pair, fp16 operands, exact diagonal)
MODES = {"f16x2": (True, True, True), "tf32x2": (True, False, True), "f16": (False, True, False), "tf32x1": (False, False, False)}


# ------------------------------------------------------------------------------------------------------ operand formats
def round_tf32(x):
    """fp32 -> tf32 with round-to-nearest (ties away), kept in fp32: what cvt.rna.tf32.f32 does on the device."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def center_round(F, shift, pair):
    """center_round_kernel: v = fp32(F - fp32(shift)), hi = tf32(v), lo = tf32(fp32(v - hi)) (pairs) or 0."""
    v = np.asarray(F, dtype=np.float32) - np.asarray(shift, dtype=np.float32)
    hi = round_tf32(v)
    lo = round_tf32(v - hi) if pair else np.zeros_like(hi)
    return hi.astype(np.float64), lo.astype(np.float64)


def fp16_pair(v, scale):
    """fp16 split of fp32 values scaled by a power of two: hi = fp16(v s), lo = fp16(v s - hi), returned unscaled."""
    vs = np.asarray(v, dtype=np.float32) * np.float32(scale)
    hi = vs.astype(np.float16)
    lo = (vs - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64) / scale, lo.astype(np.float64) / scale


def shift_estimate(F, sample_rows):
    """The generated-feature shift: fp32 of the mean of the first sample_rows rows."""
    return F[:sample_rows].mean(0).astype(np.float32).astype(np.float64)


# ------------------------------------------------------------------------------------------------------ the step algebra
def system(hi, lo, delta, lam):
    S = hi + lo
    return S.T @ S - S.shape[0] * np.outer(delta, delta) + lam * np.eye(S.shape[1])


def rhs_of(hi, lo, delta, R, lam, W_old):
    S = hi + lo
    out = S.T @ R - np.outer(delta, R.sum(0))
    return out if W_old is None else out - lam * W_old


def update_of(hi, lo, delta, R, dW):
    return R - (hi + lo) @ dW + delta @ dW


def restated_fit(F, Y, bs, num_iter, lam, shifts):
    """The fit in exact arithmetic with the shift-then-correct algebra above: block j's slab is F_j - shifts[j] (any shift),
    delta its column mean.  Returns (xs, intercept, means), the form of keystone_oracle.block_ls_fit."""
    n = F.shape[0]
    ybar = Y.mean(0)
    R = Y - ybar
    bounds = [(s, min(F.shape[1], s + bs)) for s in range(0, F.shape[1], bs)]
    xs = [np.zeros((e - s, Y.shape[1])) for s, e in bounds]
    Hs, deltas, slabs = {}, {}, {}
    for it in range(num_iter):
        for j, (s, e) in enumerate(bounds):
            S = F[:, s:e] - shifts[j]
            if j not in Hs:
                deltas[j] = S.mean(0)
                Hs[j] = system(S, 0 * S, deltas[j], lam)
            rhs = rhs_of(S, 0 * S, deltas[j], R, lam, xs[j] if it > 0 else None)
            dW = np.linalg.solve(Hs[j], rhs)
            R = update_of(S, 0 * S, deltas[j], R, dW)
            xs[j] = xs[j] + dW
    return xs, ybar, [shifts[j] + deltas[j] for j in range(len(bounds))]


# ------------------------------------------------------------------------------------------------------ bounds
def operand_error(X, mode, scale):
    """Entrywise |X - (hi + lo)| of the device's copy of an fp32 operand (residual or increment): 2^-22 relative for the pairs,
    2^-11 for one 10-bit operand; the fp16 copies are of X * scale and lose up to 2^-25 / scale (absolute) per rounding to
    fp16's subnormal spacing."""
    pair, f16, _ = MODES[mode]
    rel = 2.0 ** -22 if pair else 2.0 ** -11
    absl = (2 if pair else 1) * 2.0 ** -25 / scale if f16 else 0.0
    return rel * np.abs(X) + absl


def acc_eps(rows, chain, passes):
    """Relative error of one fp32 tensor-core sum over `rows` rows, in chains of `chain`: one ulp (2^-23) of the partial sum per
    8-deep group, then `passes` fp32 reduce-adds per chain into the output and the fp32 store and combination of the planes."""
    chain = min(chain, rows)
    return (-(-chain // 8)) * 2.0 ** -23 + (passes * -(-rows // chain) + 4) * EPS32


def delta_bound(hi, lo):
    """fp32 column sums of hi + lo (32-row chunks, then atomics over the chunks) divided by N in fp64."""
    n = hi.shape[0]
    return (n // 32 + 48) * EPS32 * np.abs(hi + lo).sum(0) / n


def diag_bound(hi, lo):
    """The exact diagonal: an fp64 sum of (hi + lo)^2 (fma chains, fp64 atomics)."""
    return (hi.shape[0] + 64) * EPS64 * ((hi + lo) ** 2).sum(0)


def system_bound(hi, lo, delta, lam, mode, chain):
    """Entrywise bound on |H_device - system(hi, lo, delta, lam)|; with an exact diagonal (the parity mode) the diagonal's
    bound is near fp64."""
    pair, _, exact_diag = MODES[mode]
    n = hi.shape[0]
    A, L = np.abs(hi + lo), np.abs(lo)
    G = A.T @ A
    b = acc_eps(n, chain, 3 if (pair and not MODES[mode][1]) else 1) * G * (1 + 2.0 ** -9) + L.T @ L
    nd = n * np.abs(np.outer(delta, delta))
    b = b + 4 * EPS64 * (G + nd + lam)
    if exact_diag:
        np.fill_diagonal(b, diag_bound(hi, lo) + 4 * EPS64 * (np.diag(G) + np.diag(nd) + lam))
    return b


def rhs_bound(hi, lo, delta, R, lam, W_old, mode, chain, rscale):
    """Entrywise bound on |rhs_device - rhs_of(...)|: C = S^T R from the device's copy of R, the fp64 column sums of R and the
    fp64 assembly."""
    pair, f16, _ = MODES[mode]
    n = hi.shape[0]
    A, L = np.abs(hi + lo), np.abs(lo)
    aR = np.abs(R)
    eR = operand_error(R, mode, rscale)
    b = acc_eps(n, chain, 3 if (pair and not f16) else 1) * (A.T @ (aR + eR)) + A.T @ eR + L.T @ (2.0 ** -11 * aR + eR)
    b = b + (n + 8) * EPS64 * np.outer(np.abs(delta), aR.sum(0))
    if W_old is not None:
        b = b + 4 * EPS64 * lam * np.abs(W_old)
    return b + 4 * EPS64 * (A.T @ aR)


def solve_bound(H, dW):
    """Backward error of a Cholesky solve in fp64, |H dW - rhs| <= gamma_{3b+1} |L||L^T||dW| with |L||L^T|_ij <= sqrt(H_ii H_jj),
    plus the fp64 evaluation of H dW (gamma_b |H||dW|, and |H_ij| <= sqrt(H_ii H_jj))."""
    b = H.shape[0]
    d = np.sqrt(np.abs(np.diag(H)))
    return (4 * b + 4) * EPS64 * np.outer(d, d @ np.abs(dW)) * 1.01


def update_bound(hi, lo, delta, R, dW, mode, dwscale):
    """Entrywise bound on |R_after_device - update_of(...)|: the product S dW along the block (K = b) from the device's copy of
    dW, cbias = fp32 of the fp64 delta^T dW, and the fp32 epilogue (two roundings) and reduce-add."""
    pair, f16, _ = MODES[mode]
    b = hi.shape[1]
    A, L = np.abs(hi + lo), np.abs(lo)
    aW = np.abs(dW)
    eW = operand_error(dW, mode, dwscale)
    prod = A @ (aW + eW)
    cb = np.abs(delta) @ aW
    err = acc_eps(b, b, 3 if (pair and not f16) else 1) * prod + A @ eW + L @ (2.0 ** -11 * aW + eW)
    return err + EPS32 * (1 + (b + 8) * 2.0 ** -29) * cb + 3 * EPS32 * (np.abs(R) + prod + cb)


def ratio(err, bound):
    """Largest err / bound; an entry with no error has ratio 0 even where its bound is 0 (an all-zero label column)."""
    err, bound = np.broadcast_arrays(np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64))
    return float(np.max(np.where(err == 0, 0.0, err / np.where(bound == 0, 1e-300, bound))))
