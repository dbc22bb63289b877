"""CPU model of the device arithmetic of the BlockLS fit (no GPU, no library): the same algorithm as engine.cu::fit_blockls
in fp64 numpy, with each operand that the device keeps in a 10-bit-mantissa format (tf32 or fp16) rounded at the same place.

What it pins on the CPU side:
  * the error budget behind the stated GPU tolerance (rel-Frobenius(W) <= 5e-3, tests/test_gpu_parity.py): the modelled
    roundings together give ~6e-4 at this shape, the order the GPU fast mode shows, and no single
    operand dominates -- the projection operands (x, W_rf), the slab, the residual operand and the increment operand;
  * the power-of-two scaling of the fp16 mode (DESIGN.md section 6): with the device's scale rule the fp16 path has the same
    error for labels of magnitude 1e-6, 1 and 1e+5, while unscaled fp16 would underflow / overflow;
  * the rank consistency rule: the residual scale must come from the global max|R| (max-all-reduce), not the local one.
"""
import numpy as np
import pytest

from oracle import keystone_oracle as ko


def round10(x):
    """Round to a 10-bit mantissa with the fp32 exponent range (what cvt.rna.tf32.f32 produces)."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)


def to_f16(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def pow2_scale(max_abs, target):
    """engine's rule (aux_kernels.cu::pow2_scale_kernel): 2^e with max * 2^e in (target / 2, target]."""
    if not (max_abs > 0 and np.isfinite(max_abs)):
        return 1.0
    s = 2.0 ** np.floor(np.log2(target / max_abs))
    return s / 2 if max_abs * s > target else s


def problem(seed=0, n=4096, d_in=60, b=256, nb=2, k=8, gamma=0.15):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d_in)).astype(np.float32).astype(np.float64)
    params = [ko.cosine_random_features_params(d_in, b, gamma, rng) for _ in range(nb)]
    Y = ko.class_label_indicators(rng.integers(0, k, n), k)
    return X, params, Y


def model_fit(X, params, Y, lam, mode, r_scale_from=None, round_proj=True, round_slab=True, round_r=True, round_dw=True):
    """mode: 'exact' | 'tf32' | 'f16' | 'f16-unscaled'.  r_scale_from: max|R0| used for the residual scale (default: own)."""
    n = X.shape[0]
    rnd = {"exact": lambda v: v, "tf32": round10, "f16": to_f16, "f16-unscaled": to_f16}[mode]
    scaled = mode == "f16"
    ymean = Y.mean(0)
    R = Y - ymean
    sr = pow2_scale(np.abs(R).max() if r_scale_from is None else r_scale_from, 4096.0) if scaled else 1.0
    Ws = []
    for W, bias in params:
        Wf = W.astype(np.float32).astype(np.float64)
        if mode != "exact" and round_proj:
            if scaled:
                sx, sw = pow2_scale(np.abs(X).max(), 4096.0), pow2_scale(np.abs(Wf).max(), 4096.0)
                Z = (to_f16(X * sx) @ to_f16(Wf * sw).T) / (sx * sw)
            else:
                Z = rnd(X) @ rnd(Wf).T
        else:
            Z = X @ Wf.T
        F = np.cos(Z + bias)
        m = F[: min(n, 1024)].mean(0)                        # shift estimate from a sample, exactness restored by delta
        S = F - m
        if mode != "exact" and round_slab:
            S = rnd(S)
        delta = S.mean(0)
        G = S.T @ S - n * np.outer(delta, delta) + lam * np.eye(S.shape[1])
        Rop = rnd(R * sr) if (mode != "exact" and round_r) else R * sr
        C = (S.T @ Rop) / sr - n * np.outer(delta, R.mean(0))
        dW = np.linalg.solve(G, C)
        if mode != "exact" and round_dw:
            sd = pow2_scale(np.abs(dW).max(), 8192.0) if scaled else 1.0
            dWop = rnd(dW * sd) / sd
        else:
            dWop = dW
        R = R - (S @ dWop - delta @ dWop)
        Ws.append(dW)
    return np.concatenate(Ws, 0)


def relfro(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def test_exact_model_equals_oracle():
    X, params, Y = problem()
    F = np.concatenate([ko.cosine_random_features(X, W.astype(np.float32).astype(np.float64), b) for W, b in params], 1)
    xs, _, _ = ko.block_ls_fit(F, Y, 256, 1, 1.0)
    assert relfro(model_fit(X, params, Y, 1.0, "exact"), np.concatenate(xs, 0)) < 1e-9


@pytest.mark.parametrize("mode", ["tf32", "f16"])
def test_error_budget_of_the_10_bit_operand_modes(mode):
    X, params, Y = problem()
    W0 = model_fit(X, params, Y, 1.0, "exact")
    total = relfro(model_fit(X, params, Y, 1.0, mode), W0)
    parts = {
        "projection": relfro(model_fit(X, params, Y, 1.0, mode, round_slab=False, round_r=False, round_dw=False), W0),
        "slab": relfro(model_fit(X, params, Y, 1.0, mode, round_proj=False, round_r=False, round_dw=False), W0),
        "residual": relfro(model_fit(X, params, Y, 1.0, mode, round_proj=False, round_slab=False, round_dw=False), W0),
        "increment": relfro(model_fit(X, params, Y, 1.0, mode, round_proj=False, round_slab=False, round_r=False), W0),
    }
    assert total < 2e-3, (total, parts)                      # GPU tolerance is 5e-3
    assert all(0 < v < total * 1.05 for v in parts.values()), parts
    assert abs(np.sqrt(sum(v * v for v in parts.values())) - total) < 0.5 * total, (total, parts)   # they add in quadrature


def test_f16_and_tf32_modes_agree():
    X, params, Y = problem(seed=3)
    W0 = model_fit(X, params, Y, 1.0, "exact")
    e32, e16 = relfro(model_fit(X, params, Y, 1.0, "tf32"), W0), relfro(model_fit(X, params, Y, 1.0, "f16"), W0)
    assert 0.5 < e16 / e32 < 2.0, (e16, e32)               # same mantissa, same error


@pytest.mark.parametrize("scale", [1e-6, 1.0, 1e5])
def test_power_of_two_scales_make_fp16_independent_of_label_units(scale):
    X, params, Y = problem(seed=5)
    rng = np.random.default_rng(6)
    Ys = rng.standard_normal(Y.shape) * scale
    W0 = model_fit(X, params, Ys, 1.0, "exact")
    assert relfro(model_fit(X, params, Ys, 1.0, "f16"), W0) < 2e-3
    if scale != 1.0:                                         # without the scales fp16 flushes to zero / overflows
        with np.errstate(invalid="ignore", over="ignore"):
            bad = model_fit(X, params, Ys, 1.0, "f16-unscaled")
        assert not np.all(np.isfinite(bad)) or relfro(bad, W0) > 2e-2


def test_residual_scale_must_be_global_across_ranks():
    """Two row shards whose residual magnitudes differ: C = sum_r S_r^T fp16(s R_r) / s needs ONE s (max-all-reduce)."""
    rng = np.random.default_rng(7)
    S = [to_f16(rng.standard_normal((512, 64))) for _ in range(2)]
    R = [rng.standard_normal((512, 4)), rng.standard_normal((512, 4)) * 1e-3]
    exact = sum(s.T @ r for s, r in zip(S, R))
    s_glob = pow2_scale(max(np.abs(r).max() for r in R), 4096.0)
    c_glob = sum(s.T @ to_f16(r * s_glob) for s, r in zip(S, R)) / s_glob
    assert relfro(c_glob, exact) < 1e-3
    s_loc = [pow2_scale(np.abs(r).max(), 4096.0) for r in R]
    assert s_loc[0] != s_loc[1]
    c_wrong = sum(s.T @ to_f16(r * sl) for s, r, sl in zip(S, R, s_loc)) / s_loc[0]   # summed as if one scale applied
    assert relfro(c_wrong, exact) > 1.0


# ------------------------------------------------------------------------------------ split-operand mode (KS_PRECISION_F16X2)
def split16(x):
    hi = to_f16(x)
    return hi, to_f16(x - hi)


def model_fit_split(X, params, Y, lam):
    """engine.cu::fit_blockls with x2 = true: every fp16 operand as hi + lo, products hi*hi + hi*lo + lo*hi; the projection as ONE
    GEMM on operands concatenated along K ([x_hi | x_lo | x_hi] . [w_hi | w_hi | w_lo]^T), as make_feat_src builds them."""
    n = X.shape[0]
    ymean = Y.mean(0)
    R = Y - ymean
    sr = pow2_scale(np.abs(R).max(), 4096.0)
    sx = pow2_scale(np.abs(X).max(), 4096.0)
    xh, xl = split16(X * sx)
    X3 = np.concatenate([xh, xl, xh], 1)
    Ws = []
    for W, bias in params:
        Wf = W.astype(np.float32).astype(np.float64)
        sw = pow2_scale(np.abs(Wf).max(), 4096.0)
        wh, wl = split16(Wf * sw)
        W3 = np.concatenate([wh, wh, wl], 1)
        F = np.cos((X3 @ W3.T) / (sx * sw) + bias)
        S = (F - F[: min(n, 1024)].mean(0)).astype(np.float32).astype(np.float64)      # the fp32 block before the split
        sh, sl = split16(S)
        delta = (sh + sl).mean(0)
        cross = sh.T @ sl
        G = sh.T @ sh + cross + cross.T - n * np.outer(delta, delta) + lam * np.eye(S.shape[1])
        rh, rl = split16(R * sr)
        C = (sh.T @ rh + sl.T @ rh + sh.T @ rl) / sr - n * np.outer(delta, R.mean(0))
        dW = np.linalg.solve(G, C)
        sd = pow2_scale(np.abs(dW).max(), 8192.0)
        dh, dl = split16(dW * sd)
        R = R - ((sh @ dh + sl @ dh + sh @ dl) / sd - delta @ dW)
        Ws.append(dW)
    return np.concatenate(Ws, 0)


def test_split_operand_mode_reaches_fp32_class_accuracy():
    X, params, Y = problem(seed=8)
    W0 = model_fit(X, params, Y, 1.0, "exact")
    e1 = relfro(model_fit(X, params, Y, 1.0, "f16"), W0)
    e2 = relfro(model_fit_split(X, params, Y, 1.0), W0)
    assert e2 < 1e-5 and e2 < e1 / 100, (e1, e2)          # SURVEY 8(d) parity-mode target: 1e-4


def test_k_concatenation_equals_three_products():
    rng = np.random.default_rng(9)
    x, w = rng.standard_normal((50, 33)), rng.standard_normal((20, 33))
    xh, xl = split16(x)
    wh, wl = split16(w)
    lhs = np.concatenate([xh, xl, xh], 1) @ np.concatenate([wh, wh, wl], 1).T
    assert np.allclose(lhs, xh @ wh.T + xl @ wh.T + xh @ wl.T, rtol=0, atol=1e-12)
    assert np.abs(lhs - x @ w.T).max() < 1e-5 * np.abs(x @ w.T).max() + 1e-6      # vs 5e-4 relative for the single fp16 product

