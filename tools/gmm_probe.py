"""The mixture fit at the reference pipelines' shapes on one GPU: (D, K, N) = (64, 16, 1e7) (ImageNet LCS after PCA) and
(80, 256, 1e6) (VOC SIFT), on synthetic standard-normal rows.

    python tools/gmm_probe.py [--iters 5] [--scale 1.0] [--out FILE]

Each shape: GaussianMixtureModelEstimator(K, maxIterations=--iters, minClusterSize=1) with the cost stop disabled, so every fit runs
--iters EM iterations after the k-means++ start, and KMeansPlusPlusEstimator(K, --iters) likewise.  One warm-up fit, then one timed
fit; the per-phase device milliseconds come from the fit statistics (CUDA events).  Reported: seeding ms, ms per EM iteration
(E-step + statistics + M-step) and per Lloyd pass, and rates from shapes:
  * flops per iteration: 3 N K D (log-likelihoods) + 2 N (2D + 1) K (the statistics product), beside the data sheet's 67 TFLOP/s
    fp64 tensor and 34 TFLOP/s fp64 vector rates;
  * bytes per iteration: X read once by the E-step and ceil(K / 64) times by the statistics, Q (fp64) written once and read
    ceil((2D + 1) / 64) times, as a share of the H100 SXM data sheet's 3.35 TB/s;
  * seeding: K - 1 passes over X (fp32) and the fp64 distances (read and written), against the same bandwidth.
The card and its power limit are read in the same run."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
FP64_TC, FP64_VEC = 67e12, 34e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies N (a smaller run for a quick check)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "iters": a.iters}
    with ks.Context(0) as ctx:
        for D, K, N in ((64, 16, 10_000_000), (80, 256, 1_000_000)):
            N = int(N * a.scale)
            X = ctx.synthetic_normal(N, D, seed=D * 1000 + K)
            m = 2 * D + 1
            flops = 3.0 * N * K * D + 2.0 * N * m * K
            by = N * D * 4.0 * (1 + math.ceil(K / 64)) + N * K * 8.0 * (1 + math.ceil(m / 64))
            seed_by = (K - 1) * (N * D * 4.0 + 2 * N * 8.0)
            est = ks.GaussianMixtureModelEstimator(K, maxIterations=a.iters, minClusterSize=1, stopTolerance=-1e300)
            est.fit(X)
            t0 = time.perf_counter()
            est.fit(X)
            wall = time.perf_counter() - t0
            st = est.stats
            it_ms = (st["estep_ms"] + st["stats_ms"] + st["mstep_ms"]) / st["iterations"]
            km = ks.KMeansPlusPlusEstimator(K, a.iters, stopTolerance=-1e300)
            km.fit(X)
            km.fit(X)
            ks_ = km.stats
            pass_ms = (ks_["estep_ms"] + ks_["stats_ms"] + ks_["mstep_ms"]) / ks_["iterations"]
            key = f"gmm_D{D}_K{K}_N{N}"
            res[key] = {"fit_wall_ms": wall * 1e3, "iterations": st["iterations"], "seeding_ms": st["seeding_ms"], "init_ms": st["init_ms"],
                        "em_iter_ms": it_ms, "estep_ms_per_iter": st["estep_ms"] / st["iterations"],
                        "stats_ms_per_iter": st["stats_ms"] / st["iterations"], "mstep_ms_per_iter": st["mstep_ms"] / st["iterations"],
                        "kmeans_pass_ms": pass_ms, "launches": st["launches"],
                        "em_TFLOP_per_s": flops / (it_ms * 1e-3) / 1e12, "em_fp64_tc_share": flops / (it_ms * 1e-3) / FP64_TC,
                        "em_fp64_vec_share": flops / (it_ms * 1e-3) / FP64_VEC, "em_GB_per_s": by / (it_ms * 1e-3) / 1e9,
                        "em_hbm_share": by / (it_ms * 1e-3) / HBM,
                        "seeding_GB_per_s": seed_by / (st["seeding_ms"] * 1e-3) / 1e9,
                        "seeding_hbm_share": seed_by / (st["seeding_ms"] * 1e-3) / HBM}
            print(key, json.dumps(res[key]), flush=True)
            X.free()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
