"""SparseLBFGSwithL2 on text-shaped sparse data on one GPU:
  * Amazon-shaped: --rows rows (1 000 000), d = 100 000, --nnz-per-row (120) entries per row drawn from a Zipf(1.1) column
    distribution, k = 2, lambda = 0, 20 iterations (what LeastSquaresEstimator runs);
  * Newsgroups-shaped: the same with k = 20.

    python tools/sparse_lbfgs_probe.py [--rows 1000000] [--cpu-rows 100000] [--profile] [--out FILE]

Reported per workload, all generated from seed 0:
  * the upload: host clock around ctx.sparse (host checks, copies, CSC sort and work tables; it ends in a synchronise);
  * a warm-up fit of 2 iterations, then a 20-iteration fit with convergence_tol = 0, timed by device events per phase (the fit's
    stats): A P per pass, A^T R per pass (one more pass than iterations: the gradient at x_0), the recursion, the all-reduces;
  * bytes per product from the shapes: 12 B per entry (int32 index, fp64 value) for the product's pass over its copy, 32 B per
    chunk of the work table, the N x k fp64 operand or result, and the d x k fp64 operand or result once; GB/s and the share of
    the H100 SXM data sheet's 3.35 TB/s;
  * the per-iteration time of the fp64 CPU restatement, scipy.sparse A @ P and A.T @ R, on a --cpu-rows row subsample at the same
    d and k, scaled to --rows rows: a stand-in for the reference's per-iteration gradient on one host (SURVEY section 8d).
--profile adds a torch.profiler run of one 2-iteration fit that lists its kernels.  The card and its power limit are read in the
same run."""
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


def make_csr(rng, n, d, per_row):
    p = 1.0 / np.arange(1, d + 1) ** 1.1
    cdf = np.cumsum(p / p.sum())
    nnz = n * per_row
    indices = np.minimum(np.searchsorted(cdf, rng.random(nnz)), d - 1).astype(np.int32)
    data = rng.standard_normal(nnz)
    indptr = np.arange(n + 1, dtype=np.int64) * per_row
    return indptr, indices, data


def chunks(lengths, bound=256):
    return int(np.maximum(1, (lengths + bound - 1) // bound).sum())


def _kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.device_time_total > 0:
            kern[ev.key] = kern.get(ev.key, 0.0) + ev.device_time_total / 1e3
    return kern


def cpu_iteration_s(indptr, indices, data, n_sub, k, rng):
    import scipy.sparse as sp
    nnz = int(indptr[n_sub])
    A = sp.csr_matrix((data[:nnz], indices[:nnz], indptr[:n_sub + 1]), shape=(n_sub, D))
    P = rng.standard_normal((D, k))
    R = rng.standard_normal((n_sub, k))
    A @ P
    t0 = time.perf_counter()
    for _ in range(3):
        Q = A @ P
        C = A.T @ R
    return (time.perf_counter() - t0) / 3, float(Q[0, 0] + C[0, 0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--nnz-per-row", type=int, default=120)
    ap.add_argument("--cpu-rows", type=int, default=100_000)
    ap.add_argument("--iterations", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "rows": a.rows, "d": D, "nnz_per_row": a.nnz_per_row, "iterations": a.iterations, "nproc": os.cpu_count()}
    rng = np.random.default_rng(0)
    t0 = time.perf_counter()
    indptr, indices, data = make_csr(rng, a.rows, D, a.nnz_per_row)
    nnz = int(indptr[-1])
    col_len = np.bincount(indices, minlength=D)
    res["generate_s"] = time.perf_counter() - t0
    res["largest_column_nnz"] = int(col_len.max())
    res["empty_columns"] = int((col_len == 0).sum())
    print("generated", json.dumps({k: res[k] for k in ("generate_s", "largest_column_nnz", "empty_columns")}), flush=True)
    row_chunks = chunks(np.diff(indptr))
    col_chunks = chunks(col_len)
    with ks.Context(0) as ctx:
        t0 = time.perf_counter()
        A = ctx.sparse((indptr, indices, data, D))
        res["upload_s"] = time.perf_counter() - t0
        print("upload_s", res["upload_s"], flush=True)
        for name, k in (("amazon", 2), ("newsgroups", 20)):
            y = ctx.labels_from_classes(rng.integers(0, k, a.rows).astype(np.int32), k)
            ks.SparseLBFGSwithL2(num_iterations=2, convergence_tol=0.0, ctx=ctx).fit(A, y)   # warm-up
            est = ks.SparseLBFGSwithL2(num_iterations=a.iterations, convergence_tol=0.0, ctx=ctx)
            est.fit(A, y)
            st = est.stats
            it = st["iterations"]
            ap_ms, atr_ms = st["ap_ms"] / it, st["atr_ms"] / (it + 1)
            by_ap = 12 * nnz + 32 * row_chunks + 8 * a.rows * k + 8 * (D + 1) * k
            by_atr = 12 * nnz + 32 * col_chunks + 8 * a.rows * k + 8 * D * k
            r = {"k": k, "iterations": it, "total_ms": st["total_ms"], "ms_per_iteration": st["total_ms"] / it,
                 "ap_ms": ap_ms, "atr_ms": atr_ms, "recursion_ms": st["solve_ms"] / it, "other_ms": st["other_ms"] / it,
                 "allreduce_ms": st["allreduce_ms"] / it,
                 "ap_GB_per_s": by_ap / ap_ms / 1e6, "ap_hbm_share": by_ap / (ap_ms * 1e-3) / HBM,
                 "atr_GB_per_s": by_atr / atr_ms / 1e6, "atr_hbm_share": by_atr / (atr_ms * 1e-3) / HBM,
                 "ap_MB": by_ap / 1e6, "atr_MB": by_atr / 1e6, "launches": st["launches"], "loss_last": st["loss_history"][-1]}
            cpu_s, _ = cpu_iteration_s(indptr, indices, data, min(a.cpu_rows, a.rows), k, rng)
            r["cpu_standin_ms_per_iteration"] = cpu_s * 1e3 * a.rows / min(a.cpu_rows, a.rows)
            res[name] = r
            print(name, json.dumps(r), flush=True)
            if a.profile:
                res[f"kernels_{name}_ms"] = _kernels(
                    lambda: ks.SparseLBFGSwithL2(num_iterations=2, convergence_tol=0.0, ctx=ctx).fit(A, y))
                print("kernels", json.dumps(res[f"kernels_{name}_ms"]), flush=True)
            y.free()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
