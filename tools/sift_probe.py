"""PixelScaler -> GrayScaler -> SIFTExtractor on VOC-shaped images on one GPU:
  * shapes 375 x 500 and 500 x 375 (x = rows; VOC's landscape and portrait images), --batch images of one shape per call;
  * settings VOC (3, 4, 4, scaleStep 0, VOCSIFTFisher.scala) and the class defaults (3, 4, 4, 1).

    python tools/sift_probe.py [--batch 64] [--reps 5] [--profile] [--out FILE]

Each case: one warm-up call, then --reps timed calls (host clock around the call; every call ends in a stream synchronise); the
median is reported, for the gray conversion (PixelScaler + GrayScaler, fused) and for SIFTExtractor.  Rates come from shapes: the
bytes the extractor must move per image are its gray pixels read once per scale, per scale 8 orientation planes of fp32 written and
read back twice, and the nKP x 128 fp32 descriptors written; GB/s is that over the time, and its share of the H100 SXM data sheet's
3.35 TB/s.  --profile adds a separate torch.profiler run that splits one SIFT call into its kernels.  The card and its power limit
are read in the same run."""
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


def _median_time(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def sift_bytes(se, x_dim, y_dim):
    npx = x_dim * y_dim
    counts = se.keypoints_per_scale(x_dim, y_dim)
    active = sum(1 for c in counts if c > 0)
    return active * (npx * 4 + 3 * 8 * npx * 4) + sum(counts) * 128 * 4


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
            gray_node, pix = ks.GrayScaler(), ks.PixelScaler()
            t_gray = _median_time(lambda: gray_node.apply(pix.apply(imgs)), a.reps)
            gray = gray_node.apply(pix.apply(imgs))
            by_gray = a.batch * x_dim * y_dim * 4 * 4
            res[f"gray_{x_dim}x{y_dim}"] = {"ms": t_gray * 1e3, "GB_per_s": by_gray / t_gray / 1e9}
            print(f"gray {x_dim}x{y_dim}", json.dumps(res[f"gray_{x_dim}x{y_dim}"]), flush=True)
            for name, params in (("voc", (3, 4, 4, 0)), ("default", (3, 4, 4, 1))):
                se = ks.SIFTExtractor(*params)
                t = _median_time(lambda: se.apply(gray), a.reps)
                by = a.batch * sift_bytes(se, x_dim, y_dim)
                key = f"sift_{name}_{x_dim}x{y_dim}"
                res[key] = {"ms": t * 1e3, "ms_per_image": t * 1e3 / a.batch, "images_per_s": a.batch / t,
                            "keypoints_per_image": se.keypoints(x_dim, y_dim), "MB_per_image": by / a.batch / 1e6,
                            "GB_per_s": by / t / 1e9, "hbm_share": by / t / HBM}
                print(key, json.dumps(res[key]), flush=True)
            if a.profile:
                import torch
                from torch.profiler import ProfilerActivity, profile
                se = ks.SIFTExtractor(3, 4, 4, 0)
                se.apply(gray)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    se.apply(gray)
                    torch.cuda.synchronize()
                kern = {}
                for ev in prof.key_averages():
                    if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.device_time_total > 0:
                        kern[ev.key] = kern.get(ev.key, 0.0) + ev.device_time_total / 1e3
                res[f"kernels_voc_{x_dim}x{y_dim}_ms"] = kern
                print("kernels", json.dumps(kern), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
