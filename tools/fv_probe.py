"""The LCS Fisher-vector branch at the reference pipelines' shapes on one GPU:
  * lcs   LCSExtractor(4, 16, 6) on 256 x 256 x 3 images, batches of --batch images (ImageNetSiftLcsFV's settings)
  * fv    FisherVector at (D, K, n) = (64, 16, 3136) (ImageNet LCS after PCA) and (80, 256, 3136) (VOC), --batch items of n descriptors
  * tail  NormalizeRows -> SignedHellingerMapper -> NormalizeRows on the (80, 256) Fisher vectors

    python tools/fv_probe.py [--batch 256] [--reps 5] [--out FILE]

Each case: one warm-up call, then --reps timed calls (host clock around the call; every call ends in a stream synchronise); the
median is reported.  Rates are computed from shapes:
  * lcs: images/s, and the bytes every image must move (its fp32 pixels in, its nKP x 96 fp32 descriptors out) over the time, as a
    share of the H100 SXM data sheet's 3.35 TB/s;
  * fv: fp64 flops 3 n K D (posterior: difference, square, fused multiply-add) + 2 n (2D + 1) K (the statistics product) over the time,
    beside the data sheet's 67 TFLOP/s fp64 tensor and 34 TFLOP/s fp64 vector rates; bytes: descriptors read twice, posteriors
    written and read in fp64, the output written;
  * tail: 2 x 4 bytes per element and pass, three passes.
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
FP64_TC, FP64_VEC = 67e12, 34e12


def _median_time(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "batch": a.batch, "reps": a.reps}
    rng = np.random.default_rng(0)
    with ks.Context(0) as ctx:
        # ---- LCS
        imgs = ks.ImageBatch.from_images(ctx, rng.integers(0, 256, (a.batch, 256, 256, 3)).astype(np.float32))
        lcs = ks.LCSExtractor(4, 16, 6)
        t = _median_time(lambda: lcs.apply(imgs), a.reps)
        nkp = lcs.keypoints(256, 256)
        by = a.batch * (256 * 256 * 3 * 4 + nkp * 96 * 4)
        res["lcs"] = {"ms": t * 1e3, "images_per_s": a.batch / t, "GB_per_s": by / t / 1e9, "hbm_share": by / t / HBM}
        print("lcs", json.dumps(res["lcs"]), flush=True)
        # ---- Fisher vectors
        n = 3136
        offs = np.arange(a.batch + 1, dtype=np.int64) * n
        last = None
        for D, K in ((64, 16), (80, 256)):
            means, variances = rng.standard_normal((D, K)) * 0.3, rng.uniform(0.5, 2.0, (D, K))
            gmm = ks.GaussianMixtureModel(means, variances, np.full(K, 1.0 / K), ctx=ctx)
            batch = ks.ItemBatch(ctx.synthetic_normal(a.batch * n, D, seed=D * 1000 + K), offs)
            fv = ks.FisherVector(gmm)
            t = _median_time(lambda: fv.apply(batch), a.reps)
            N = a.batch * n
            flops = 3.0 * N * K * D + 2.0 * N * (2 * D + 1) * K
            by = 2.0 * N * D * 4 + 2.0 * N * K * 8 + a.batch * 2.0 * D * K * 4
            key = f"fv_D{D}_K{K}"
            res[key] = {"ms": t * 1e3, "items_per_s": a.batch / t, "TFLOP_per_s": flops / t / 1e12, "fp64_tc_share": flops / t / FP64_TC,
                        "fp64_vec_share": flops / t / FP64_VEC, "GB_per_s": by / t / 1e9, "hbm_share": by / t / HBM}
            print(key, json.dumps(res[key]), flush=True)
            last = fv.apply(batch)
        # ---- normalisation tail on the (80, 256) vectors
        tail = ks.Pipeline([ks.NormalizeRows(), ks.SignedHellingerMapper(), ks.NormalizeRows()])
        t = _median_time(lambda: tail(last), a.reps)
        by = 3 * 2.0 * last.rows * last.cols * 4
        res["tail"] = {"ms": t * 1e3, "items_per_s": last.rows / t, "GB_per_s": by / t / 1e9, "hbm_share": by / t / HBM}
        print("tail", json.dumps(res["tail"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
