"""A/B timing of engine options inside ONE process on the config-3 workload (GPU box): options are switched with
ks_ctx_set_option between fits, every configuration gets 1 warm-up + 3 timed fits, and the list is run twice so that
drift (clocks, temperature) shows up as a difference between the two passes instead of as a fake effect."""
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
import keystone_b200 as ks


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    rng = np.random.default_rng(0)
    d_in, n_out, nrf, k = 440, 4096, 16, 1000
    X = rng.standard_normal((n, d_in), dtype=np.float32)
    cls = rng.integers(0, k, n).astype(np.int32)
    with ks.Context(0) as ctx:
        x = ctx.matrix(X)
        y = ctx.labels_from_classes(cls, k)
        rfs = [ks.CosineRandomFeatures.create(ctx, d_in, n_out, 0.0555, rng) for _ in range(nrf)]
        feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
        est = ks.BlockLeastSquaresEstimator(n_out, 1, 1.0, precision="f16")
        # (proj_f16, gram_chunk_rows) -- chunk 0 = the engine's own choice
        configs = [(1, 0), (0, 0), (1, 4096)]
        if len(sys.argv) > 2:
            configs = [tuple(int(v) for v in c.split(",")) for c in sys.argv[2:]]
        for rep in range(2):
            for proj, chunk in configs:
                ctx.set_option("proj_f16", proj)
                ctx.set_option("gram_chunk_rows", chunk)
                est.fit(feats, y)
                ts = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    est.fit(feats, y)
                    ts.append(1e3 * (time.perf_counter() - t0))
                st = ctx.last_fit_stats()
                print(json.dumps({"probe": "ab_fit", "pass": rep, "proj_f16": proj, "chunk_rows": chunk,
                                  "ms": [round(t, 1) for t in ts], "featurize_ms": st["featurize_ms"], "gram_ms": st["gram_ms"],
                                  "update_ms": st["update_ms"], "solve_ms": st["solve_ms"]}), flush=True)


if __name__ == "__main__":
    main()
