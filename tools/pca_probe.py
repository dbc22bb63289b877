"""PCA, ZCA whitening and approximate PCA at the reference pipelines' shapes on one GPU:
  * zca      ZCA 100 000 x 108 (the CIFAR whitener of RandomPatchCifar)
  * voc      PCA 1e6 x 128 -> 80 (VOCSIFTFisher)
  * imagenet PCA 1e7 x 128 -> 64 (ImageNetSiftLcsFV)
  * wide     PCA 1e6 x 4096 -> 256
  * approx   ApproximatePCA 200 000 x 16 384 -> 100 (q = 10, p = 5)

    python tools/pca_probe.py [--only zca,voc,imagenet,wide,approx] [--reps 3] [--sub 20000] [--out FILE]

Data are N(0.5, 1) rows generated on the device.  Per shape: one warm-up fit, then --reps timed fits (host clock around the
synchronous fit) with the median's phase split from the fit statistics.  Rates:
  * gram: the algorithmic N d^2 flops of the symmetric covariance Gram (its upper tiles) over gram_ms, as a share of the H100 SXM
    data sheet's 67 TFLOP/s fp64 tensor rate;
  * skinny (approx only): the (q + 1) X-products Y = X B read N d fp32 and write N l fp64 each, over skinny_ms, as a share of
    3.35 TB/s.
Parity: the same fit on the first --sub rows against the fp64 oracle (tests/pca_oracle.py).  The card and its power limit are read
first."""
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

SHAPES = {
    "zca": ("zca", 100_000, 108, 0),
    "voc": ("pca", 1_000_000, 128, 80),
    "imagenet": ("pca", 10_000_000, 128, 64),
    "wide": ("pca", 1_000_000, 4096, 256),
    "approx": ("approx", 200_000, 16_384, 100),
}


def _estimator(ks, ctx, kind, dims):
    if kind == "zca":
        return lambda x: ks.ZCAWhitenerEstimator(0.1, ctx=ctx).fit_single(x)
    if kind == "pca":
        return lambda x: ks.PCAEstimator(dims, ctx=ctx).fit(x)
    return lambda x: ks.ApproximatePCAEstimator(dims, q=10, p=5, ctx=ctx).fit(x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=",".join(SHAPES))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sub", type=int, default=20000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks
    import pca_oracle as po

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "runs": []}
    ctx = ks.Context(0)
    for name in a.only.split(","):
        kind, n, d, dims = SHAPES[name]
        x = ctx.synthetic_normal(n, d, seed=7, mean=0.5)
        fit = _estimator(ks, ctx, kind, dims)
        fit(x)  # warm-up
        walls, stats = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            m = fit(x)
            walls.append(time.perf_counter() - t0)
            stats.append(ctx.last_fit_stats())
            del m
        i = int(np.argsort(walls)[len(walls) // 2])
        st = {k: v for k, v in stats[i].items() if k not in ("eigenvalues", "singular_values")}
        out = {"shape": name, "kind": kind, "n": n, "d": d, "dims": dims, "wall_s": walls, "stats": st}
        if kind != "approx":
            out["gram_tflops"] = n * d * d / (st["gram_ms"] * 1e-3) / 1e12
            out["gram_share_of_67tf"] = out["gram_tflops"] / 67.0
        else:
            l, q = dims + 5, 10
            byts = (q + 1) * (n * d * 4.0 + n * l * 8.0)
            out["skinny_tb_s"] = byts / (st["skinny_ms"] * 1e-3) / 1e12
            out["skinny_share_of_3_35tb"] = out["skinny_tb_s"] / 3.35
        # parity on a row subsample, fitted the same way
        del x
        sub = min(a.sub if kind != "approx" else a.sub // 5, n)
        Xs = ctx.synthetic_normal(sub, d, seed=7, mean=0.5)  # counter-based: the first sub rows of the timed data
        Xh = Xs.to_numpy(np.float32).astype(np.float64)
        m = fit(Xs)
        if kind == "zca":
            Wr, mr = po.zca_fit(Xh, 0.1)
            out["parity_rel_fro_whitener"] = float(np.linalg.norm(m.whitener - Wr) / np.linalg.norm(Wr))
        elif kind == "pca":
            out["parity_max_abs_pca_mat"] = float(np.abs(m.pca_mat - po.compute_pca(Xh, dims)).max())
        else:
            ref = po.approximate_pca(Xh, po.omega(d, dims + 5, 0), dims, 10)
            out["parity_max_abs_pca_mat"] = float(np.abs(m.pca_mat - ref).max())
        out["parity_rows"] = sub
        del m, Xs
        print(json.dumps(out), flush=True)
        res["runs"].append(out)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
