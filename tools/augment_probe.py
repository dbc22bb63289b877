"""The CIFAR random-patch front end and test-time augmentation at CIFAR size on one GPU: 50 000 seeded 32 x 32 x 3 byte images,
RandomPatcher(10, 24, 24) + RandomImageTransformer(0.5, flip) = 500 000 training views, CenterCornerPatcher(24, 24, true) on 10 000
test images = 100 000 test views.

    python tools/augment_probe.py [--images 50000] [--test-images 10000] [--filters 100,1600] [--reps 3] [--out FILE]

Every device call ends in a stream synchronise; times are host clocks around the call (median of --reps after a warm-up).  Rates
come from shapes:
  ks_image_views   each output value read once from the source and written once (4 + 4 B per value);
  scaler           fit: two passes over the fp32 features (8 B per value), apply: read + write (8 B per value);
and their share of the H100 SXM data sheet's 3.35 TB/s.  The Convolver is timed over the views and over their materialised matrix
(whose size is reported; the gather that made it is not in that time).  The per-stage times of random_patch_cifar_augmented run
the pipeline's stages one by one.  The card and its power limit are read in the same run.  --out FILE also writes the JSON there."""
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


def _timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=50000)
    ap.add_argument("--test-images", type=int, default=10000)
    ap.add_argument("--filters", default="100,1600")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import keystone_b200 as ks
    from keystone_b200 import pipelines as P

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    res = {"card": card, "images": a.images, "test_images": a.test_images, "reps": a.reps}
    rng = np.random.default_rng(0)
    labels = rng.integers(0, 10, a.images).astype(np.int32)
    data = rng.integers(0, 256, (a.images, 3, 32, 32)).astype(np.uint8)
    test_labels = rng.integers(0, 10, a.test_images).astype(np.int32)
    test_data = rng.integers(0, 256, (a.test_images, 3, 32, 32)).astype(np.uint8)
    with ks.Context(0) as ctx:
        images = P._train_images(ctx, data)
        views, t_tables = _timed(lambda: ks.RandomImageTransformer(0.5, ks.flip_horizontal).apply(ks.RandomPatcher(10, 24, 24).apply(images)))
        res["view_tables_host_s"] = t_tables
        n_views = views.rows

        def gather():
            views._matrix = None
            return views.matrix
        t = _median_time(gather, a.reps)
        vals = n_views * 24 * 24 * 3
        res["image_views"] = {"views": n_views, "s": t, "GBps": 8 * vals / t / 1e9, "hbm_share": 8 * vals / t / HBM}
        print("image_views", res["image_views"], flush=True)
        mat = views.matrix

        filt = np.random.default_rng(1).standard_normal((100, 108))
        conv = ks.Convolver(ctx, filt, 24, 24, 3, whitener_means=np.zeros(108))
        chain = lambda x: ks.ImageVectorizer().apply(ks.Pooler(9, 10).apply(ks.SymmetricRectifier(alpha=0.25).apply(conv.apply(x))))
        conv_res = {name: {"s": _median_time(lambda: chain(src), a.reps)} for name, src in (("views", views), ("materialised", mat))}
        conv_res["materialised_views_GB"] = mat.rows * 24 * 24 * 3 * 4 / 1e9
        res["convolver_100_filters"] = conv_res
        print("convolver", conv_res, flush=True)
        del mat
        views._matrix = None

        feats = chain(views)
        vals = feats.rows * feats.cols
        t_fit = _median_time(lambda: ks.StandardScaler().fit(feats), a.reps)
        model = ks.StandardScaler().fit(feats)
        t_apply = _median_time(lambda: model.apply(feats), a.reps)
        res["scaler"] = {"rows": feats.rows, "cols": feats.cols, "fit_s": t_fit, "fit_GBps": 8 * vals / t_fit / 1e9,
                         "fit_hbm_share": 8 * vals / t_fit / HBM, "apply_s": t_apply, "apply_GBps": 8 * vals / t_apply / 1e9,
                         "apply_hbm_share": 8 * vals / t_apply / HBM}
        print("scaler", res["scaler"], flush=True)
        del feats

        n_test = a.test_images * 10
        scores = ctx.matrix(np.random.default_rng(2).standard_normal((n_test, 10)).astype(np.float32))
        names = np.repeat(np.arange(a.test_images), 10)
        tl = np.repeat(test_labels, 10)
        res["evaluator"] = {policy: {"views": n_test, "s": _median_time(
            lambda: ks.AugmentedExamplesEvaluator(names, 10, policy).evaluate(scores, tl), a.reps)} for policy in ("average", "borda")}
        print("evaluator", res["evaluator"], flush=True)

        res["pipeline"] = {}
        for nf in [int(v) for v in a.filters.split(",") if v]:
            st = {}
            try:
                conf = P.RandomCifarFeaturizerConfig(numFilters=nf, lam=10.0)
                (filters, W, means), st["learn_filters_s"] = _timed(lambda: P.learn_filters(ctx, images, conf))
                conv_n = ks.Convolver(ctx, filters, 24, 24, 3, whitener_means=means)
                rect, pool = ks.SymmetricRectifier(alpha=conf.alpha), ks.Pooler(conf.poolStride, conf.poolSize)
                raw, st["featurize_train_s"] = _timed(lambda: ks.ImageVectorizer().apply(pool.apply(rect.apply(conv_n.apply(views)))))
                scaler, st["scaler_fit_s"] = _timed(lambda: ks.StandardScaler().fit(raw))
                F, st["scaler_apply_s"] = _timed(lambda: scaler.apply(raw))
                del raw
                y = ctx.labels_from_classes(np.repeat(labels, 10), 10)
                model, st["block_ls_fit_s"] = _timed(lambda: ks.BlockLeastSquaresEstimator(4096, 1, conf.lam).fit(F, y))
                del F, y
                test_views = ks.CenterCornerPatcher(24, 24, True).apply(P._train_images(ctx, test_data))
                fitted = P.RandomPatchCifarModel(conv_n, rect, pool, scaler, model, filters, W, means)
                s, st["test_featurize_apply_s"] = _timed(lambda: fitted.apply(test_views))
                m, st["evaluate_s"] = _timed(lambda: ks.AugmentedExamplesEvaluator(names, 10).evaluate(s, tl))
                st["features"] = nf * 2 * 4
                st["test_accuracy_on_noise"] = float(np.trace(m.confusionMatrix) / m.confusionMatrix.sum())
                del s, fitted, model, test_views, conv_n
            except Exception as e:  # report what ran; a shape that does not fit on the card is a finding, not a crash
                st["error"] = repr(e)[:400]
            res["pipeline"][str(nf)] = st
            print("pipeline", nf, st, flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
