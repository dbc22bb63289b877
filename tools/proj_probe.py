"""The projection (feature generation) kernels alone at the benchmark's shape: N = 1M rows, d_in = 440, one 4096-column block.

    python tools/proj_probe.py [--n 1000000] [--iters 5] [--out FILE]

For the parity mode's fp16 pair (with the exact diagonal) and the fast mode's fp16 slab, ks_debug_time_slab times the block fit's
first-sweep produce_slab launch (CUDA events, after a warm-up launch, on the look-ahead stream with its reserved SMs).  The EPI_RBF
rate comes from the generation phase of one kernel ridge regression fit at N = 200 000, d = 440, blocks of 4096 (tools/krr_probe.py
has the whole fit).  Prints the card name, power limit and the median SM clock sampled while the kernels ran, in the same call."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _smi(query):
    return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()


class ClockSampler:
    def __init__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.wait(0.2):
            try:
                self.samples.append(float(_smi("clocks.sm")))
            except ValueError:
                pass

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def median(self):
        return statistics.median(self.samples) if self.samples else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=440)
    ap.add_argument("--b", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--krr-n", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks
    from keystone_b200._capi import KS_PRECISION_F16, KS_PRECISION_F16X2, check, lib

    res = {"card": _smi("name"), "power_limit_w": _smi("power.limit"), "n": a.n, "d_in": a.d, "b": a.b}
    rng = np.random.default_rng(0)
    ctx = ks.Context(0)
    x = ctx.synthetic_normal(a.n, a.d, seed=3, mean=0.0, stddev=1.0)
    rf = ks.CosineRandomFeatures(ctx, rng.standard_normal((a.b, a.d)) * 0.1, rng.random(a.b) * 2 * np.pi)
    arr = (C.c_int64 * 1)(rf.handle)
    kinds = {"parity_pair": (KS_PRECISION_F16X2, 0, 3), "fast_f16": (KS_PRECISION_F16, 1, 1)}
    with ClockSampler() as clk:
        for name, (prec, round_out, products) in kinds.items():
            ms = C.c_double()
            check(ctx.handle, lib().ks_debug_time_slab(ctx.handle, x.handle, arr, 1, prec, round_out, a.b, a.iters, C.byref(ms),
                                                       None, None, None))
            mma_flops = products * 2.0 * a.n * a.d * a.b            # executed: hi hi + lo hi + hi lo for the pair
            slab_bytes = (4 if prec == KS_PRECISION_F16X2 else 2) * a.n * a.b
            res[name] = {"ms": ms.value, "mma_tflops": mma_flops / (ms.value * 1e-3) / 1e12,
                         "slab_gb_per_s": slab_bytes / (ms.value * 1e-3) / 1e9}
            print(name, json.dumps(res[name]), flush=True)
        del x
        # EPI_RBF: the generation phase of a kernel ridge regression fit (fp16 pair of the Gaussian kernel block)
        Xk = ctx.synthetic_normal(a.krr_n, a.d, seed=7, mean=0.5, stddev=1.0)
        Yk = ctx.labels_from_classes(rng.integers(0, 147, a.krr_n), 147)
        est = ks.KernelRidgeRegression(ks.GaussianKernelGenerator(1.0 / (2 * a.d)), 1e-1, a.b, 1, ctx=ctx)
        est.fit(Xk, Yk)  # warm-up
        est.fit(Xk, Yk)
        st = ctx.last_fit_stats()
        res["rbf_generate"] = {"ms": st["generate_ms"], "mma_tflops": st["generate_mma_flops"] / (st["generate_ms"] * 1e-3) / 1e12}
        print("rbf_generate", json.dumps(res["rbf_generate"]), flush=True)
    res["median_sm_clock_mhz"] = clk.median()
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
