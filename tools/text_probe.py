"""Times the text front end (DESIGN.md section 23) on a seeded synthetic corpus: each phase of the Amazon reviews featurizer, the
hashing path and the whole Amazon pipeline, plus a CPU stand-in (the exact host oracle of tests/text_oracle.py on a subsample,
scaled up; it is a stand-in for a host implementation, not the reference).  The upload is timed in two parts, the host UTF-8 encode
and the device upload with its UTF-8 check, after one untimed full-size upload.

    python tools/text_probe.py [--docs 1000000] [--vocab 200000] [--cpu-docs 10000] [--out result.json]

Corpus: log-normal document lengths around 120 tokens, Zipf(1.1) over ``--vocab`` synthetic words (every 13th word non-ASCII,
every 5th capitalised), 10 % of words followed by punctuation.  Timing: every library call ends in a synchronise of the library's
own stream, so a host clock around a call (after a context synchronise) measures the device work plus launch overhead; the library
exposes no events on that stream.
"""
from __future__ import annotations

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


def corpus(n_docs: int, vocab: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    words = []
    for i in range(vocab):
        w = "w%x" % i
        if i % 13 == 0:
            w = "é" + w + "ß"
        if i % 5 == 0:
            w = w.capitalize()
        words.append(w)
    words = np.array(words, dtype=object)
    lens = np.maximum(1, rng.lognormal(np.log(120), 0.5, n_docs).astype(np.int64))
    total = int(lens.sum())
    ids = np.minimum(rng.zipf(1.1, total) - 1, vocab - 1)
    punct = np.array(["", "", "", "", "", "", "", "", "", ".", ",", "!", "?", ")"], dtype=object)
    toks = words[ids] + punct[rng.integers(0, len(punct), total)]
    labels = (rng.random(n_docs) < 0.5).astype(np.int32)
    docs, p = [], 0
    for n in lens.tolist():
        docs.append(" ".join(toks[p:p + n]))
        p += n
    return docs, labels


def timed(ctx, fn):
    ctx.synchronize()
    t = time.perf_counter()
    out = fn()
    ctx.synchronize()
    return out, time.perf_counter() - t


def array_size(ctx, handle, which) -> int:
    import ctypes as C
    from keystone_b200 import _capi
    n = C.c_int64(0)
    _capi.check(ctx.handle, _capi.lib().ks_text_array_size(ctx.handle, handle, which, C.byref(n)))
    return n.value


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip()
        return q.splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--vocab", type=int, default=200_000)
    ap.add_argument("--cpu-docs", type=int, default=10_000)
    ap.add_argument("--features", type=int, default=100_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import keystone_b200 as ks
    from keystone_b200 import _capi, pipelines
    from keystone_b200.loaders import LabeledData
    import text_oracle as to

    t0 = time.perf_counter()
    docs, labels = corpus(a.docs, a.vocab)
    gen_s = time.perf_counter() - t0
    n_bytes = sum(len(d.encode()) for d in docs)
    res = {"card": card(), "docs": a.docs, "vocab": a.vocab, "text_bytes": n_bytes, "corpus_generation_s": gen_s}
    with ks.Context(0) as ctx:
        # warm-up of every kernel on a small batch
        small = ks.TermFrequency(lambda x: 1.0).apply(ks.NGramsFeaturizer([1, 2]).apply(
            ks.Tokenizer().apply(ks.LowerCase().apply(ks.Trim(ctx=ctx).apply(docs[:1000])))))
        ks.CommonSparseFeatures(1000).fit(small).apply(small)
        ks.NGramsHashingTF([1, 2], 1 << 20).apply(small.tokens)

        import ctypes as C
        from keystone_b200.context import TextBatch, _encode_all

        def upload(data, off):
            h = C.c_int64(0)
            _capi.check(ctx.handle, _capi.lib().ks_text_from_host(ctx.handle, data.ctypes.data_as(C.c_void_p), data.shape[0],
                                                                  off.ctypes.data_as(C.c_void_p), off.shape[0] - 1, C.byref(h)))
            return TextBatch(ctx, h.value, off.shape[0] - 1)

        (data, off), res["host_encode_s"] = timed(ctx, lambda: _encode_all(docs, "document"))
        upload(data, off).free()                                   # warm-up at full size (memory pool, pinned staging)
        text, res["device_upload_s"] = timed(ctx, lambda: upload(data, off))
        del data, off
        res["upload_s"] = res["host_encode_s"] + res["device_upload_s"]
        toks, res["trim_lower_tokenize_s"] = timed(ctx, lambda: ks.Tokenizer().apply(ks.LowerCase().apply(ks.Trim().apply(text))))
        tf, res["ngrams_tf_s"] = timed(ctx, lambda: ks.TermFrequency(lambda x: 1.0).apply(ks.NGramsFeaturizer([1, 2]).apply(toks)))
        vec, res["common_sparse_features_fit_s"] = timed(ctx, lambda: ks.CommonSparseFeatures(a.features).fit(tf))
        sm, res["vectorize_s"] = timed(ctx, lambda: vec.apply(tf))
        hsm, res["ngrams_hashing_tf_s"] = timed(ctx, lambda: ks.NGramsHashingTF([1, 2], 1 << 20).apply(toks))
        n_tok = array_size(ctx, toks.handle, _capi.KS_TEXT_TOKEN_BEGIN)
        res.update({"tokens": n_tok, "tf_entries": array_size(ctx, tf.handle, _capi.KS_TEXT_TERM_ORDER), "csr_nnz": int(sm.nnz),
                    "hashing_nnz": int(hsm.nnz)})
        del text, toks, tf, vec, sm, hsm
        front = res["upload_s"] + res["trim_lower_tokenize_s"] + res["ngrams_tf_s"] + res["common_sparse_features_fit_s"] + res["vectorize_s"]
        res["front_end_s"] = front
        res["text_GBps_front_end"] = n_bytes / front / 1e9
        device = front - res["upload_s"]
        res["device_phases_s"] = device
        res["text_GBps_device_phases"] = n_bytes / device / 1e9
        res["tokens_per_s_front_end"] = n_tok / front
        res["csr_entries_per_s_front_end"] = res["csr_nnz"] / front
        n_train = int(a.docs * 0.9)
        _, res["amazon_pipeline_s"] = timed(ctx, lambda: pipelines.amazon_reviews_pipeline(
            ctx, LabeledData(labels[:n_train], docs[:n_train]), LabeledData(labels[n_train:], docs[n_train:]),
            pipelines.AmazonReviewsConfig(commonFeatures=a.features)))
    # the CPU stand-in: the exact host oracle, one thread, on a subsample, scaled by bytes
    sub = docs[:a.cpu_docs]
    sub_bytes = sum(len(d.encode()) for d in sub)
    t = time.perf_counter()
    tfs = to.text_features(sub, 2)
    space = to.common_sparse_features(tfs, a.features)
    to.vectorize(space, tfs)
    cpu = time.perf_counter() - t
    res["cpu_standin_docs"] = len(sub)
    res["cpu_standin_s_measured"] = cpu
    res["cpu_standin_s_scaled"] = cpu * n_bytes / sub_bytes
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
