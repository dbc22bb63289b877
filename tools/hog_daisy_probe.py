"""HogExtractor and DaisyExtractor on VOC-shaped images on one GPU:
  * shapes 375 x 500 and 500 x 375 (x = rows; VOC's landscape and portrait images), --batch images of one shape per call;
  * HOG at bins 5 and 16 after PixelScaler (bin 8 rounds both sides of a VOC image up, where the reference reads past the end of
    the image, so the node rejects it), DAISY at the class defaults after GrayScaler.

    python tools/hog_daisy_probe.py [--batch 64] [--reps 5] [--profile] [--out FILE]

Each case: one warm-up call, then --reps timed calls (host clock around the call; every call ends in a stream synchronise); the
median is reported.  Rates come from shapes, counting each buffer once per pass that must touch it:
  HOG    the 3-channel fp32 image read once, the fp64 magnitude and 1-byte orientation of every visible pixel written and read back,
         the fp32 histograms written and read twice, and the (cells x 32) fp32 features written;
  DAISY  the fp32 gray image read; per fp64 plane of the image: ix and iy (two passes: 2 written, 2 read, 2 written, then 2 read by
         the orientation pass), H written by it, 2H for its pass along y, 4H for each further layer; the fp32 descriptors written.
GB/s is that over the time, and its share of the H100 SXM data sheet's 3.35 TB/s.  --profile adds a torch.profiler run that splits
one call of each node into its kernels.  The card and its power limit are read in the same run."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def _median_time(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def hog_bytes(x_dim, y_dim, bin_):
    nx, ny = (int(math.floor(d / bin_ + 0.5)) for d in (x_dim, y_dim))
    rows = max(nx - 2, 0) * max(ny - 2, 0)
    return x_dim * y_dim * 3 * 4 + 2 * 9 * (nx * bin_) * (ny * bin_) + 3 * 18 * nx * ny * 4 + rows * 32 * 4


def daisy_bytes(de, x_dim, y_dim):
    npx = x_dim * y_dim
    H, Q = de.daisyH, de.daisyQ
    planes = 8 + H + 2 * H + 4 * H * (Q - 1)
    return npx * 4 + planes * npx * 8 + de.keypoints(x_dim, y_dim) * de.daisyFeatureSize * 4


def _kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.device_time_total > 0:
            kern[ev.key] = kern.get(ev.key, 0.0) + ev.device_time_total / 1e3
    return kern


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "batch": a.batch, "reps": a.reps}
    rng = np.random.default_rng(0)
    with ks.Context(0) as ctx:
        for (x_dim, y_dim) in ((375, 500), (500, 375)):
            imgs = ks.ImageBatch.from_images(ctx, rng.integers(0, 256, (a.batch, x_dim, y_dim, 3)).astype(np.float32))
            scaled = ks.PixelScaler().apply(imgs)
            gray = ks.GrayScaler().apply(imgs)
            cases = [(f"hog{b}", ks.HogExtractor(b), scaled, hog_bytes(x_dim, y_dim, b)) for b in (5, 16)]
            de = ks.DaisyExtractor()
            cases.append(("daisy", de, gray, daisy_bytes(de, x_dim, y_dim)))
            for name, node, data, per_image in cases:
                t = _median_time(lambda: node.apply(data), a.reps)
                by = a.batch * per_image
                key = f"{name}_{x_dim}x{y_dim}"
                res[key] = {"ms": t * 1e3, "ms_per_image": t * 1e3 / a.batch, "images_per_s": a.batch / t,
                            "MB_per_image": per_image / 1e6, "GB_per_s": by / t / 1e9, "hbm_share": by / t / HBM}
                print(key, json.dumps(res[key]), flush=True)
                if a.profile:
                    res[f"kernels_{key}_ms"] = _kernels(lambda: node.apply(data))
                    print("kernels", json.dumps(res[f"kernels_{key}_ms"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
