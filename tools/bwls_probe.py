"""BlockWeightedLeastSquaresEstimator on one GPU against the fp64 oracle, at the C5 configuration in miniature and on the
separated-classes problem of tests/test_gpu_bwls.py (the same generators):
  * c5: class-sorted rows with Zipf class sizes, d_in = 440 -> 2 x 1024 cosine features (generated on the fly), k = 147,
        lambda = 6e-5, w = 0.25, b = 1024, one sweep; --rows scales it up (default 64 000);
  * separated: 50 000 materialised rows x 256 features, 20 classes with centroids 1.5 sigma apart per coordinate and a common
        offset of 50, lambda = 1e-2, w = 0.25, b = 256, two sweeps.

    python tools/bwls_probe.py [--rows 64000] [--only c5,separated] [--out FILE]

Per problem and precision mode ("default" = the tf32-pair parity mode, "tf32"): rel-Fro(W) against the oracle, the fit time
(device events, after a warm-up fit) and the fit statistics, as JSON lines.  The card and its power limit are read first."""
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


def _run(ctx, ks, ko, name, data, F, cls, k, bs, iters, lam, w, res):
    t0 = time.perf_counter()
    xs, fb = ko.bwls_fit(F, ko.class_label_indicators(cls, k), bs, iters, lam, w)
    oracle_s = time.perf_counter() - t0
    Wr = np.concatenate(xs, 0)
    y = ctx.labels_from_classes(cls, k)
    for prec in ("default", "tf32"):
        est = ks.BlockWeightedLeastSquaresEstimator(bs, iters, lam, w, precision=prec)
        est.fit(data, y)  # warm-up
        m = est.fit(data, y)
        st = ctx.last_fit_stats()
        Wg = np.concatenate(m.xs, 0)
        out = {"problem": name, "precision": prec, "n": len(cls), "d": F.shape[1], "k": k, "block_size": bs, "num_iter": iters,
               "lam": lam, "w": w, "rel_fro_W": float(np.linalg.norm(Wg - Wr) / np.linalg.norm(Wr)),
               "b_max_abs_err": float(np.abs(m.b_opt - fb).max()), "fit_ms": st["total_ms"], "oracle_s": oracle_s, "stats": st}
        print(json.dumps(out), flush=True)
        res["runs"].append(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=64000)
    ap.add_argument("--only", default="c5,separated")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks
    import test_gpu_bwls as T
    from oracle import keystone_oracle as ko

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "runs": []}
    only = set(a.only.split(","))
    ctx = ks.Context(0)
    if "c5" in only:
        c5 = T.C5
        rng = np.random.default_rng(147)
        cls = np.repeat(np.arange(c5["k"]), T.zipf_sizes(a.rows, c5["k"], rng))
        X, params, F = T.cosine_problem(rng, cls, c5["k"], c5["d_in"], c5["nrf"], c5["n_out"], 0.1)
        _run(ctx, ks, ko, f"c5-mini-{a.rows}", T.generated(ctx, X, params), F, cls, c5["k"], c5["bs"], 1, c5["lam"], c5["w"], res)
        del X, F
    if "separated" in only:
        rng = np.random.default_rng(50)
        cls = np.repeat(np.arange(20), T.zipf_sizes(50000, 20, rng))
        F32 = T.gaussian_classes(rng, cls, 256, 20, sep=1.5, offset=50.0)
        _run(ctx, ks, ko, "separated-50000", ctx.matrix(F32), F32.astype(np.float64), cls, 20, 256, 2, 1e-2, 0.25, res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
