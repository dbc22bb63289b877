"""Dense L-BFGS against the block solver on one GPU, in the same call:
  * N = 1M rows of x_in (d_in = 440) -> D = 16 384 (4 cosine maps of 4096), k = 10 and k = 147;
  * a materialised 50 000 x 160 000 CIFAR-shaped matrix at k = 10 (skipped when it does not fit beside the slabs).

    python tools/lbfgs_probe.py [--iters 20] [--precision default] [--only gen10,gen147,cifar10] [--out FILE]

Per shape: DenseLBFGSwithL2(num_iterations = iters, convergence_tol = 0, reg_param = lam) after a warm-up fit, its time per
iteration and phase split, the algorithmic rate (4 N D k per iteration, plus 2 x 2 N d_in D for the two projections of
generated features), BlockLeastSquaresEstimator(4096, 1, N lam) on the same data, the block solver's training loss in the
L-BFGS objective and the first L-BFGS iteration that reaches it.  For the k = 10 generated shape also rel-Fro(W) against the
fp64 oracle (tests/lbfgs_oracle.py) on a row subsample fitted the same way.  The card and its power limit are read first."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _loss(pred, Y, W, lam):
    """f = |A_c W - Y_c|^2 / (2N) + lam / 2 |W|^2 of a centred model: its predictions are A_c W + ybar."""
    return float(((pred - Y) ** 2).sum() / (2 * Y.shape[0]) + lam / 2 * (W ** 2).sum())


def _run(ctx, ks, name, feats, y, Y, n, D, k, d_in, lam, a, res):
    out = {"shape": name, "n": n, "d": D, "k": k, "lam": lam}
    est = ks.DenseLBFGSwithL2(num_iterations=a.iters, convergence_tol=0.0, reg_param=lam, ctx=ctx, precision=a.precision)
    est.fit(feats, y)  # warm-up
    t0 = time.perf_counter()
    m = est.fit(feats, y)
    out["lbfgs_wall_s"] = time.perf_counter() - t0
    st = dict(est.stats)
    hist = st.pop("loss_history")
    it = max(1, st["iterations"])
    out["lbfgs_stats"] = st
    out["lbfgs_ms_per_iter"] = st["total_ms"] / it
    per_iter_flops = 4.0 * n * D * k + (4.0 * n * d_in * D if d_in else 0.0)
    out["lbfgs_algorithmic_tflops"] = per_iter_flops / (out["lbfgs_ms_per_iter"] * 1e-3) / 1e12
    out["lbfgs_loss_history"] = hist
    del m
    bl = ks.BlockLeastSquaresEstimator(4096, 1, n * lam, ctx=ctx, precision=a.precision)
    bl.fit(feats, y)  # warm-up
    t0 = time.perf_counter()
    mb = bl.fit(feats, y)
    out["block_wall_s"] = time.perf_counter() - t0
    sb = ctx.last_fit_stats()
    out["block_total_ms"] = sb["total_ms"]
    Wb = np.concatenate(mb.xs, 0)
    out["block_train_loss"] = _loss(mb.apply(feats).to_numpy(np.float32).astype(np.float64), Y, Wb, lam)
    reach = [i for i, f in enumerate(hist) if f <= out["block_train_loss"]]
    out["lbfgs_iters_to_block_loss"] = reach[0] if reach else None
    del mb
    print(json.dumps({kk: v for kk, v in out.items() if kk != "lbfgs_loss_history"}), flush=True)
    res["runs"].append(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--precision", default="default")
    ap.add_argument("--only", default="gen10,gen147,cifar10")
    ap.add_argument("--sub", type=int, default=8192)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks
    import lbfgs_oracle as lo
    from oracle import keystone_oracle as ko

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "iters": a.iters, "precision": a.precision, "runs": []}
    only = set(a.only.split(","))
    ctx = ks.Context(0)
    n, d_in, maps, lam = 1_000_000, 440, 4, 1e-4
    rng = np.random.default_rng(0)
    params = [ko.cosine_random_features_params(d_in, 4096, 1.0 / np.sqrt(d_in), rng) for _ in range(maps)]
    x = ctx.synthetic_normal(n, d_in, seed=3)
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
    for k in (10, 147):
        if f"gen{k}" not in only:
            continue
        cls = rng.integers(0, k, n)
        y = ctx.labels_from_classes(cls, k)
        _run(ctx, ks, f"generated-1M-x-16384-k{k}", feats, y, y.to_numpy(), n, 4096 * maps, k, d_in, lam, a, res)
        if k == 10:  # accuracy on a row subsample against the fp64 oracle
            Xs = x.to_numpy()[: a.sub]
            Ys = y.to_numpy()[: a.sub]
            xs_ = ctx.matrix(Xs.astype(np.float32))
            fs = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(xs_)
            est = ks.DenseLBFGSwithL2(num_iterations=a.iters, convergence_tol=0.0, reg_param=lam, ctx=ctx, precision=a.precision)
            Wg = np.concatenate(est.fit(fs, ctx.matrix(Ys.astype(np.float32))).xs, 0)
            F = np.concatenate([ko.cosine_random_features(Xs, W, b) for W, b in params], 1)
            Wr = lo.fit(F, Ys, True, 10, 0.0, a.iters, lam)[0]
            res["subsample"] = {"rows": a.sub, "rel_fro_W": float(np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr))}
            print(json.dumps(res["subsample"]), flush=True)
    del feats, rfs, x
    if "cifar10" in only:
        nc, dc, k = 50_000, 160_000, 10
        try:
            A = ctx.synthetic_normal(nc, dc, seed=5, mean=0.2)
            cls = rng.integers(0, k, nc)
            y = ctx.labels_from_classes(cls, k)
            _run(ctx, ks, "materialised-50000-x-160000-k10", A, y, y.to_numpy(), nc, dc, k, 0, 1e-3, a, res)
        except ks.KeystoneError as e:
            res["cifar10_skipped"] = str(e)
            print("cifar10 skipped:", e, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
