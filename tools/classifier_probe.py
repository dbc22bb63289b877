"""LogisticRegressionEstimator and NaiveBayesEstimator at text-pipeline sizes on one GPU:
  * logistic regression, Amazon-shaped: --rows rows (1 000 000), d = 100 000, --nnz-per-row (120) entries per row from a Zipf(1.1)
    column distribution, k = 2, --iterations (20) iterations (AmazonReviewsPipeline's numIters);
  * the same at k = 20;
  * naive Bayes, Newsgroups-shaped: the same matrix, k = 20;
  * dense logistic regression: --dense-rows rows (1 000 000) of d = 4096 fp32 features, k = 10.

    python tools/classifier_probe.py [--rows 1000000] [--dense-rows 1000000] [--cpu-rows 100000] [--out FILE]

The sparse values are non-negative (term-frequency-like) so one matrix serves both fits; labels are uniform class ids from seed 0
(random labels: the timings, not the models, are the point).  Reported per workload:
  * a warm-up fit (2 iterations), then the timed fit with convergence_tol = 0: device events per phase from the fit's stats, per
    iteration: A P, A^T R (one more pass than iterations: the gradient at W_0), the line search (its trial kernels and all-reduces),
    the softmax/residual pass, the recursion, the all-reduces; the line-search evaluations of each iteration;
  * bytes per product from the shapes (sparse: 12 B per entry and 32 B per work-table chunk of the product's copy, the N x (k-1)
    fp64 operand or result and the d x (k-1) fp64 operand or result; dense: the 4 N d bytes of the features plus both fp64 sides),
    GB/s and the share of the H100 SXM data sheet's 3.35 TB/s;
  * a CPU stand-in labelled as such: scipy / numpy fp64 A @ P and A.T @ R on a --cpu-rows subsample, scaled to the full rows.
The card and its power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
D = 100_000
D_DENSE = 4096


def make_csr(rng, n, d, per_row):
    p = 1.0 / np.arange(1, d + 1) ** 1.1
    cdf = np.cumsum(p / p.sum())
    nnz = n * per_row
    indices = np.minimum(np.searchsorted(cdf, rng.random(nnz)), d - 1).astype(np.int32)
    data = rng.random(nnz) + 0.5
    indptr = np.arange(n + 1, dtype=np.int64) * per_row
    return indptr, indices, data


def chunks(lengths, bound=256):
    return int(np.maximum(1, (lengths + bound - 1) // bound).sum())


def per_iteration(st):
    it = max(st["iterations"], 1)
    return {"iterations": st["iterations"], "stop_reason": st["stop_reason"], "total_ms": st["total_ms"],
            "ms_per_iteration": st["total_ms"] / it, "ap_ms": st["ap_ms"] / it, "atr_ms": st["atr_ms"] / (it + 1),
            "line_search_ms": st["line_search_ms"] / it, "softmax_ms": st["softmax_ms"] / (it + 1),
            "recursion_ms": st["recursion_ms"] / it, "allreduce_ms": st["allreduce_ms"] / it,
            "line_search_evals": st["line_search_evals"], "launches": st["launches"], "loss_first_last": [st["loss_history"][0],
                                                                                                          st["loss_history"][-1]]}


def bandwidth(r, by_ap, by_atr):
    r.update({"ap_MB": by_ap / 1e6, "atr_MB": by_atr / 1e6, "ap_GB_per_s": by_ap / r["ap_ms"] / 1e6, "atr_GB_per_s": by_atr / r["atr_ms"] / 1e6,
              "ap_hbm_share": by_ap / (r["ap_ms"] * 1e-3) / HBM, "atr_hbm_share": by_atr / (r["atr_ms"] * 1e-3) / HBM})


def cpu_standin_ms(A, n_full, kk, rng):
    """fp64 A @ P and A.T @ R on the subsample A (scipy.sparse or numpy), per iteration, scaled to n_full rows."""
    P = rng.standard_normal((A.shape[1], kk))
    R = rng.standard_normal((A.shape[0], kk))
    A @ P
    t0 = time.perf_counter()
    for _ in range(3):
        A @ P
        A.T @ R
    return (time.perf_counter() - t0) / 3 * 1e3 * n_full / A.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dense-rows", type=int, default=1_000_000)
    ap.add_argument("--nnz-per-row", type=int, default=120)
    ap.add_argument("--cpu-rows", type=int, default=100_000)
    ap.add_argument("--iterations", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import scipy.sparse as sp

    import keystone_b200 as ks

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "rows": a.rows, "d": D, "nnz_per_row": a.nnz_per_row, "iterations": a.iterations, "nproc": os.cpu_count(),
           "cpu_standin": "scipy/numpy fp64 A @ P + A.T @ R on a subsample, scaled; not the reference's code"}
    rng = np.random.default_rng(0)
    indptr, indices, data = make_csr(rng, a.rows, D, a.nnz_per_row)
    nnz = int(indptr[-1])
    row_chunks = chunks(np.diff(indptr))
    col_chunks = chunks(np.bincount(indices, minlength=D))
    n_sub = min(a.cpu_rows, a.rows)
    A_sub = sp.csr_matrix((data[:int(indptr[n_sub])], indices[:int(indptr[n_sub])], indptr[:n_sub + 1]), shape=(n_sub, D))
    with ks.Context(0) as ctx:
        A = ctx.sparse((indptr, indices, data, D))
        for name, k in (("logistic_k2", 2), ("logistic_k20", 20)):
            kk = k - 1
            y = rng.integers(0, k, a.rows).astype(np.int32)
            ks.LogisticRegressionEstimator(k, num_iters=2, convergence_tol=0.0, ctx=ctx).fit(A, y)   # warm-up
            est = ks.LogisticRegressionEstimator(k, num_iters=a.iterations, convergence_tol=0.0, ctx=ctx)
            est.fit(A, y)
            r = per_iteration(est.stats)
            bandwidth(r, 12 * nnz + 32 * row_chunks + 8 * a.rows * kk + 8 * D * kk, 12 * nnz + 32 * col_chunks + 8 * a.rows * kk + 8 * D * kk)
            r["cpu_standin_ms_per_iteration"] = cpu_standin_ms(A_sub, a.rows, kk, rng)
            res[name] = r
            print(name, json.dumps(r), flush=True)
        k = 20
        y = rng.integers(0, k, a.rows).astype(np.int32)
        ks.NaiveBayesEstimator(k, ctx=ctx).fit(A, y)   # warm-up
        t0 = time.perf_counter()
        nb = ks.NaiveBayesEstimator(k, ctx=ctx)
        nb.fit(A, y)
        st = nb.stats
        by = 12 * nnz + 32 * col_chunks + 8 * a.rows * k + 8 * D * k
        r = {"k": k, "host_s": time.perf_counter() - t0, "total_ms": st["total_ms"], "product_ms": st["products_ms"],
             "finish_ms": st["finish_ms"], "other_ms": st["other_ms"], "product_MB": by / 1e6,
             "product_GB_per_s": by / st["products_ms"] / 1e6, "product_hbm_share": by / (st["products_ms"] * 1e-3) / HBM}
        Y = np.zeros((n_sub, k))
        Y[np.arange(n_sub), y[:n_sub]] = 1.0
        t0 = time.perf_counter()
        A_sub.T @ Y
        r["cpu_standin_ms"] = (time.perf_counter() - t0) * 1e3 * a.rows / n_sub
        res["naive_bayes_k20"] = r
        print("naive_bayes_k20", json.dumps(r), flush=True)
        A.free()

        # dense: 1M x 4096 fp32 generated on the device, k = 10
        k, kk = 10, 9
        X = ctx.synthetic_normal(a.dense_rows, D_DENSE, 1, 0, 0.0, 1.0 / np.sqrt(D_DENSE))
        y = rng.integers(0, k, a.dense_rows).astype(np.int32)
        ks.LogisticRegressionEstimator(k, num_iters=2, convergence_tol=0.0, ctx=ctx).fit(X, y)
        est = ks.LogisticRegressionEstimator(k, num_iters=a.iterations, convergence_tol=0.0, ctx=ctx)
        est.fit(X, y)
        r = per_iteration(est.stats)
        by = 4 * a.dense_rows * D_DENSE + 8 * a.dense_rows * kk + 8 * D_DENSE * kk
        bandwidth(r, by, by)
        r["flops_per_product"] = 2.0 * a.dense_rows * D_DENSE * kk
        Xs = np.random.default_rng(1).standard_normal((min(a.cpu_rows, 20000), D_DENSE)) / np.sqrt(D_DENSE)
        r["cpu_standin_ms_per_iteration"] = cpu_standin_ms(Xs, a.dense_rows, kk, rng)
        res["dense_logistic_k10"] = r
        print("dense_logistic_k10", json.dumps(r), flush=True)
        X.free()
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
