"""Kernel ridge regression at TIMIT dimensions on one GPU: N = 200 000 training rows, d = 440, k = 147 classes, block size 4096,
one epoch (48 full blocks and a 3392-row tail).

    python tools/krr_probe.py [--n 200000] [--runs 3] [--out FILE]

Prints the card and its power limit, the fit time of each run after a warm-up fit, the per-phase times of the last run, the
achieved rate of the generation GEMM (executed MMA flops over its event time; the 989 TFLOP/s fp16 data-sheet figure is a
ceiling, not a target) and rel-Fro(W) against the fp64 oracle on an 8192-row subsample fitted the same way."""
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

FP16_PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense fp16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--d", type=int, default=440)
    ap.add_argument("--k", type=int, default=147)
    ap.add_argument("--block", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--sub", type=int, default=8192)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks
    import krr_oracle as ko

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    rng = np.random.default_rng(0)
    gamma, lam = 1.0 / (2 * a.d), 1e-1
    ctx = ks.Context(0)
    X = ctx.synthetic_normal(a.n, a.d, seed=7, mean=0.5, stddev=1.0)   # uncentred inputs: the kernel object shifts them
    cls = rng.integers(0, a.k, a.n)
    Y = ctx.labels_from_classes(cls, a.k)
    est = ks.KernelRidgeRegression(ks.GaussianKernelGenerator(gamma), lam, a.block, 1, ctx=ctx)
    res = {"card": card, "n": a.n, "d": a.d, "k": a.k, "block_size": a.block, "epochs": 1}
    est.fit(X, Y)  # warm-up
    times = []
    for _ in range(a.runs):
        t0 = time.perf_counter()
        m = est.fit(X, Y)
        times.append(time.perf_counter() - t0)
        st = ctx.last_fit_stats()
        del m
    res["fit_s"] = times
    res["stats_last_run"] = st
    res["generate_tflops"] = st["generate_mma_flops"] / (st["generate_ms"] * 1e-3) / 1e12
    res["generate_share_of_fp16_datasheet_ceiling"] = res["generate_tflops"] / FP16_PEAK_TFLOPS
    print(json.dumps(res), flush=True)

    # accuracy on a subsample, same settings
    Xs = X.to_numpy()[: a.sub]
    Ys = Y.to_numpy()[: a.sub]
    ms = est.fit(ctx.matrix(Xs.astype(np.float32)), ctx.matrix(Ys.astype(np.float32)))
    W = np.concatenate(ms.xs, 0)
    Wr = np.concatenate(ko.krr_fit(Xs, Ys, gamma, lam, a.block, 1), 0)
    res["subsample_rows"] = a.sub
    res["subsample_rel_fro_W"] = float(np.linalg.norm(W - Wr) / np.linalg.norm(Wr))
    print(json.dumps({"subsample_rows": a.sub, "rel_fro_W": res["subsample_rel_fro_W"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
