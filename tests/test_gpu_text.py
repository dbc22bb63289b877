"""The text front end on the device (DESIGN.md section 23) against the exact host oracle tests/text_oracle.py: every comparison is
exact (strings, token lists, CSR arrays, feature spaces).  The reference suites run through the nodes (T/ = src/test/scala/keystoneml/:
nodes/nlp/{StringUtilsSuite,NGramSuite,HashingTFSuite,NGramsHashingTFSuite}, nodes/misc/{TermFrequencySuite,
SparseFeatureVectorizerSuite}), then edge documents, collisions, rejections and both text pipelines in miniature."""
import math
import random

import numpy as np
import pytest

import text_oracle as to

pytestmark = pytest.mark.gpu

STRINGS = ["  The quick BROWN fo.X ", " ! !.,)JumpeD. ovER the LAZy DOG.. ! "]
DATUM = "this sentence is a sentence is the some there some then there some".split(" ")
EDGE = ["", "   ", "...", ".a.", "a..b", " x", "İstanbul ΟΔΟΣ Ⱥ", "smile \U0001F600 \U00010400 ok", "tab\tsep\x0bv\x0cf",
        "non breaking", "MiXeD-CaSe, punct!!! (yes)", "ends with sep ...", " em space"]


@pytest.fixture(scope="module")
def ctx():
    import keystone_b200 as ks
    c = ks.Context(0)
    yield c
    c.close()


def _csr_equal(sm, ref):
    got = sm.to_csr()
    for g, r in zip(got, ref):
        assert np.array_equal(g, r), (g, r)


def _pipeline_strings(docs):
    return [to.tokenize(to.lower(to.trim(d))) for d in docs]


def test_string_utils_suite(ctx):
    import keystone_b200 as ks
    assert ks.Trim(ctx=ctx).apply(STRINGS).to_host() == ["The quick BROWN fo.X", "! !.,)JumpeD. ovER the LAZy DOG.. !"]
    assert ks.LowerCase(ctx=ctx).apply(STRINGS).to_host() == ["  the quick brown fo.x ", " ! !.,)jumped. over the lazy dog.. ! "]
    assert ks.Tokenizer(ctx=ctx).apply(STRINGS).to_host() == [["", "The", "quick", "BROWN", "fo", "X"],
                                                              ["", "JumpeD", "ovER", "the", "LAZy", "DOG"]]


def test_edge_documents_and_unicode(ctx):
    import keystone_b200 as ks
    t = ctx.text(EDGE)
    assert t.to_host() == EDGE
    trimmed = ks.Trim().apply(t)
    lowered = ks.LowerCase().apply(trimmed)
    assert trimmed.to_host() == [to.trim(d) for d in EDGE]
    assert lowered.to_host() == [to.lower(to.trim(d)) for d in EDGE]
    assert ks.Tokenizer().apply(t).to_host() == [to.tokenize(d) for d in EDGE]
    toks = ks.Tokenizer().apply(lowered)
    assert toks.to_host() == _pipeline_strings(EDGE)
    flat = [w for d in _pipeline_strings(EDGE) for w in d]
    assert toks.java_hashes().tolist() == [to.java_hash(w) for w in flat]


def test_lowercase_table_every_code_point(ctx):
    import keystone_b200 as ks
    cps = [c for c in range(0x110000) if not 0xD800 <= c < 0xE000]
    docs = ["".join(chr(c) for c in cps[i:i + 4096]) for i in range(0, len(cps), 4096)]
    assert ks.LowerCase(ctx=ctx).apply(docs).to_host() == [to.lower(d) for d in docs]


def test_hash_values(ctx):
    import keystone_b200 as ks
    toks = ks.Tokenizer(ctx=ctx).apply(["hello Seq \U0001F600"])
    assert toks.java_hashes().tolist() == [99162322, 83007, 1772899]


def test_large_document_next_to_empty_ones(ctx):
    import keystone_b200 as ks
    rng = random.Random(5)
    words = ["Alpha", "beta", "GAMMA", "delta", "épée", "Ωmega", "x"]
    big = " ".join(rng.choice(words) + rng.choice(["", ",", ".", "!"]) for _ in range(36000))
    assert len(big.encode()) > 200_000
    docs = [""] * 50 + [big] + ["", "   ", "z"] * 20
    toks = ks.Tokenizer().apply(ks.LowerCase().apply(ks.Trim(ctx=ctx).apply(docs)))
    ref = _pipeline_strings(docs)
    assert toks.to_host() == ref
    tf = ks.TermFrequency().apply(ks.NGramsFeaturizer([1, 2, 3]).apply(toks))
    assert tf.to_host() == [to.term_frequency(to.ngrams(d, [1, 2, 3])) for d in ref]


def test_ngram_suite_and_short_documents(ctx):
    import keystone_b200 as ks
    docs = ["Pipelines are awesome", "NLP is awesome"]
    toks = ks.Tokenizer(ctx=ctx).apply(docs)
    assert ks.NGramsFeaturizer([1]).apply(toks).to_host() == [[("Pipelines",), ("are",), ("awesome",)], [("NLP",), ("is",), ("awesome",)]]
    assert ks.NGramsFeaturizer(range(2, 4)).apply(toks).to_host() == [
        [("Pipelines", "are"), ("Pipelines", "are", "awesome"), ("are", "awesome")],
        [("NLP", "is"), ("NLP", "is", "awesome"), ("is", "awesome")]]
    assert ks.NGramsFeaturizer([6]).apply(toks).to_host() == [[], []]
    short = ["one", "two words", "", "three words here", "..."]
    st = ks.Tokenizer(ctx=ctx).apply(short)
    ref = [to.tokenize(d) for d in short]
    for orders in ([1], [1, 2], [2, 3], [3, 4], [4]):
        tf = ks.TermFrequency().apply(ks.NGramsFeaturizer(orders).apply(st))
        assert tf.to_host() == [to.term_frequency(to.ngrams(d, orders)) for d in ref]
        _csr_equal(ks.HashingTF(1000).apply(ks.NGramsFeaturizer(orders).apply(st)), to.hashing_tf([to.ngrams(d, orders) for d in ref], 1000))


def test_term_frequency_suite(ctx):
    import keystone_b200 as ks
    data = [["b", "a", "c", "b", "b", "a", "b"]]
    assert ks.TermFrequency(ctx=ctx).apply(data).to_host() == [[("b", 4.0), ("a", 2.0), ("c", 1.0)]]
    log = ks.TermFrequency(lambda x: math.log(x + 1), ctx=ctx).apply(data).to_host()
    assert log == [to.term_frequency(data[0], lambda x: math.log(x + 1))]


def test_hashing_tf_suites(ctx):
    import keystone_b200 as ks
    datum = ["1", "2", "4", "4", "4", "4", "2"]
    for dims in (4000, 2):
        _csr_equal(ks.HashingTF(dims, ctx=ctx).apply([datum]), to.hashing_tf([datum], dims))
    toks = ctx.tokens([DATUM])
    for orders, dims in (((1, 1), 40000), ((1, 3), 40000), ((2, 3), 40000), ((1, 3), 6), ((2, 7), 97)):
        r = list(range(orders[0], orders[1] + 1))
        fused = ks.NGramsHashingTF(r, dims).apply(toks)
        chained = ks.HashingTF(dims).apply(ks.NGramsFeaturizer(r).apply(toks))
        ref = to.ngrams_hashing_tf([DATUM], r, dims)
        _csr_equal(fused, ref)
        _csr_equal(chained, ref)
        _csr_equal(chained, to.hashing_tf([to.ngrams(DATUM, r)], dims))
    a = ks.HashingTF(40000).apply(toks).to_csr()
    b = ks.HashingTF(40000).apply(ks.NGramsFeaturizer([1]).apply(toks)).to_csr()
    assert not np.array_equal(a[1], b[1])                   # String.hashCode versus seqHash of a 1-tuple


def test_sparse_feature_vectorizer_suite(ctx):
    import keystone_b200 as ks
    test = [[("Third", 4.0), ("Fourth", 6.0), ("First", 1.0)]]
    v = ks.SparseFeatureVectorizer({"First": 0, "Second": 1, "Third": 2}, ctx=ctx)
    _csr_equal(v.apply(test), to.vectorize({"First": 0, "Second": 1, "Third": 2}, test))
    train = [[("First", 0.0), ("Second", 6.0)], [("Third", 3.0), ("Second", 4.0)]]
    v = ks.AllSparseFeatures(ctx=ctx).fit(train)
    assert v.feature_space == to.all_sparse_features(train)
    _csr_equal(v.apply(test), to.vectorize(to.all_sparse_features(train), test))
    train = [[("First", 0.0), ("Second", 6.0)], [("Third", 3.0), ("Second", 4.8)], [("Third", 7.0), ("Fourth", 5.0)],
             [("Fifth", 5.0), ("Second", 7.3)]]
    v = ks.CommonSparseFeatures(2, ctx=ctx).fit(train)
    assert v.feature_space == {"Second": 0, "Third": 1}
    test = [[("Third", 4.0), ("Seventh", 8.0), ("Second", 1.3), ("Fourth", 6.0), ("First", 1.0)]]
    _csr_equal(v.apply(test), to.vectorize(v.feature_space, test))
    assert v.apply(test).to_csr()[2].tolist() == [1.3, 4.0]


def _corpus(seed, n_docs, vocab_size, mean_len=12):
    rng = random.Random(seed)
    words = ["W%d" % i if i % 7 else "mot%dé" % i for i in range(vocab_size)]
    docs = []
    for _ in range(n_docs):
        n = max(0, int(rng.lognormvariate(math.log(mean_len), 0.6)))
        docs.append(" ".join(words[min(int(rng.paretovariate(1.1)) - 1, vocab_size - 1)] + rng.choice(["", "", ",", "."])
                             for _ in range(n)))
    return docs


def test_ties_at_the_cut_and_disjoint_test_vocabulary(ctx):
    import keystone_b200 as ks
    train = ["a b c", "c d", "e f", "a f", "g"]      # counts: a 2, c 2, f 2, then b d e g 1
    tf = ks.TermFrequency().apply(ks.NGramsFeaturizer([1, 2]).apply(ks.Tokenizer(ctx=ctx).apply(train)))
    ref_tf = [to.term_frequency(to.ngrams(to.tokenize(d), [1, 2])) for d in train]
    assert tf.to_host() == ref_tf
    for k in (1, 2, 3, 4, 5, 100):
        v = ks.CommonSparseFeatures(k).fit(tf)
        assert v.feature_space == to.common_sparse_features(ref_tf, k)
        assert list(v.feature_space.values()) == list(range(min(k, len(to.all_sparse_features(ref_tf)))))
    v = ks.CommonSparseFeatures(3).fit(tf)
    test = ["x y z", "zz a", "c"]           # mostly unseen words: their token ids differ from the training batch's
    ttf = ks.TermFrequency().apply(ks.NGramsFeaturizer([1, 2]).apply(ks.Tokenizer(ctx=ctx).apply(test)))
    ref_test = [to.term_frequency(to.ngrams(to.tokenize(d), [1, 2])) for d in test]
    _csr_equal(v.apply(ttf), to.vectorize(v.feature_space, ref_test))


@pytest.mark.parametrize("bits", [64, 3, 1])
def test_forced_hash_collisions(bits):
    import keystone_b200 as ks
    c = ks.Context(0)
    try:
        if bits < 64:
            c.set_option("debug_text_hash_bits", bits)
        docs = _corpus(11, 300, 400)
        toks = ks.Tokenizer().apply(ks.LowerCase().apply(ks.Trim(ctx=c).apply(docs)))
        ref_toks = _pipeline_strings(docs)
        assert toks.to_host() == ref_toks
        tf = ks.TermFrequency().apply(ks.NGramsFeaturizer([1, 2]).apply(toks))
        ref_tf = [to.term_frequency(to.ngrams(d, [1, 2])) for d in ref_toks]
        assert tf.to_host() == ref_tf
        v = ks.CommonSparseFeatures(150).fit(tf)
        assert v.feature_space == to.common_sparse_features(ref_tf, 150)
        assert ks.AllSparseFeatures().fit(tf).feature_space == to.all_sparse_features(ref_tf)
        test = _corpus(12, 100, 600)
        ttf = ks.TermFrequency().apply(ks.NGramsFeaturizer([1, 2]).apply(ks.Tokenizer().apply(ks.LowerCase().apply(ks.Trim(ctx=c).apply(test)))))
        _csr_equal(v.apply(ttf), to.vectorize(v.feature_space, [to.term_frequency(to.ngrams(d, [1, 2])) for d in _pipeline_strings(test)]))
        host_space = ks.SparseFeatureVectorizer(v.feature_space, ctx=c)
        _csr_equal(host_space.apply(ttf), v.apply(ttf).to_csr())
    finally:
        c.close()


def test_reruns_are_bit_identical(ctx):
    import keystone_b200 as ks
    docs = _corpus(21, 500, 300)

    def run():
        tf = ks.TermFrequency().apply(ks.NGramsFeaturizer([1, 2, 3]).apply(ks.Tokenizer().apply(ks.LowerCase().apply(ks.Trim(ctx=ctx).apply(docs)))))
        sp = ks.CommonSparseFeatures(200).fit(tf)
        return tf.to_host(), sp.feature_space, sp.apply(tf).to_csr(), ks.NGramsHashingTF([1, 2], 1 << 20).apply(tf.tokens).to_csr()

    a, b = run(), run()
    assert a[0] == b[0] and a[1] == b[1]
    for x, y in list(zip(a[2], b[2])) + list(zip(a[3], b[3])):
        assert np.array_equal(x, y)


def test_rejections(ctx):
    import keystone_b200 as ks
    with pytest.raises(ValueError):
        ks.NGramsFeaturizer([0, 1])
    with pytest.raises(ValueError):
        ks.NGramsFeaturizer([1, 3])
    with pytest.raises(ValueError):
        ks.NGramsHashingTF([2, 1], 10)
    with pytest.raises(ValueError):
        ks.Tokenizer(sep="\\s+")
    for loc in ("tr", "tr_TR", "az", "lt-LT"):
        with pytest.raises(ValueError):
            ks.LowerCase(loc)
    ks.LowerCase("en_US")
    toks = ks.Tokenizer(ctx=ctx).apply(["a b c d e f"])
    with pytest.raises(ks.KeystoneError, match="above 4"):
        ks.TermFrequency().apply(ks.NGramsFeaturizer([1, 2, 3, 4, 5]).apply(toks))
    assert ks.NGramsHashingTF([1, 2, 3, 4, 5], 50).apply(toks).nnz > 0
    with pytest.raises(ks.KeystoneError, match="UTF-8"):
        ctx.text([b"ok", b"bad \xff byte"])
    with pytest.raises(ks.KeystoneError, match="UTF-8"):
        ctx.text([b"split \xc3", b"\xa9 across documents"])
    with pytest.raises(ks.KeystoneError, match="UTF-8"):
        ctx.text([b"overlong \xc0\xaf"])
    with pytest.raises(ks.KeystoneError, match="surrogate"):
        ctx.text(["lone \ud800 surrogate"])
    with pytest.raises(ks.KeystoneError, match="not finite"):
        ks.TermFrequency(lambda x: math.inf if x > 1 else 1.0).apply(ctx.tokens([["a", "a"]]))
    with pytest.raises(ks.KeystoneError, match="not finite"):
        ks.TermFrequency(lambda x: float("nan")).apply(ctx.tokens([["a"]]))


def test_multi_rank_fit_is_rejected_by_the_node(ctx):
    """The node's own check, on one GPU: the context object reports two ranks.  The library's check (``c.world > 1`` in
    ``ks_sparse_features_fit``) is covered by ``test_two_ranks_reject_the_fit_in_the_library``, which needs two GPUs."""
    import keystone_b200 as ks
    tf = ks.TermFrequency().apply(ks.Tokenizer(ctx=ctx).apply(["a b"]))
    ctx.world_size = 2          # what a multi-rank context reports; the fit refuses before any collective
    try:
        with pytest.raises(ks.KeystoneError, match="one rank"):
            ks.CommonSparseFeatures(5).fit(tf)
        with pytest.raises(ks.KeystoneError, match="one rank"):
            ks.AllSparseFeatures().fit(tf)
    finally:
        ctx.world_size = 1


def _two_rank_worker(rank, world, id_holder, ret):
    import ctypes as C
    import os
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    import keystone_b200 as ks
    from keystone_b200 import _capi
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    tf = ks.TermFrequency().apply(ks.Tokenizer(ctx=ctx).apply(["a b", "b c"] if rank == 0 else ["c d"]))
    h = C.c_int64(0)
    rc = _capi.lib().ks_sparse_features_fit(ctx.handle, tf.handle, 5, C.byref(h))     # the C ABI directly, past the node's check
    ret[f"rc{rank}"] = (rc, _capi.lib().ks_last_error(ctx.handle).decode())
    ret[f"hash{rank}"] = ks.HashingTF(64).apply(tf.tokens).to_csr()[1].tolist()       # row-local nodes work on any rank
    ctx.close()


def test_two_ranks_reject_the_fit_in_the_library():
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import keystone_b200 as ks
    mgr = mp.Manager()
    id_holder, ret = mgr.dict(), mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_two_rank_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    for r in (0, 1):
        rc, msg = ret[f"rc{r}"]
        assert rc == -1 and "one rank" in msg
    assert ret["hash0"] == to.hashing_tf([["a", "b"], ["b", "c"]], 64)[1].tolist()
    assert ret["hash1"] == to.hashing_tf([["c", "d"]], 64)[1].tolist()


def test_empty_spaces_host_tuples_and_repeated_terms_are_handled(ctx):
    import keystone_b200 as ks
    empty = ks.TermFrequency().apply(ks.Tokenizer(ctx=ctx).apply(["..."]))
    for est in (ks.AllSparseFeatures(), ks.CommonSparseFeatures(3)):
        with pytest.raises(ks.KeystoneError, match="at least one feature"):
            est.fit(empty)
    with pytest.raises(ks.KeystoneError, match="1 to"):
        ks.SparseFeatureVectorizer({}, ctx=ctx)
    with pytest.raises(ks.KeystoneError, match="NGramsFeaturizer"):
        ks.TermFrequency(ctx=ctx).apply([[("a", "b"), ("a", "b")]])
    with pytest.raises(ks.KeystoneError, match="NGramsFeaturizer"):
        ks.HashingTF(16, ctx=ctx).apply([[("a",)]])
    # a host batch that repeats a term within a document: one entry per column, values added in order
    v = ks.SparseFeatureVectorizer({"x": 0, ("x", "y"): 1}, ctx=ctx)
    docs = [[("x", 1.5), (("x", "y"), 2.0), ("x", 0.25)], [("z", 1.0)], [(("x", "y"), 4.0), (("x", "y"), -1.0)]]
    _csr_equal(v.apply(docs), to.vectorize({"x": 0, ("x", "y"): 1}, docs))


def test_hash_bits_option_is_fixed_once_text_exists():
    import keystone_b200 as ks
    c = ks.Context(0)
    try:
        c.set_option("debug_text_hash_bits", 8)
        t = c.text(["a"])
        with pytest.raises(ks.KeystoneError, match="before any text object"):
            c.set_option("debug_text_hash_bits", 4)
        del t
        c.set_option("debug_text_hash_bits", 4)      # allowed again once no text object is left
    finally:
        c.close()


def _labelled_corpus(seed, n, k):
    rng = random.Random(seed)
    vocab = ["w%d" % i for i in range(800)]
    topics = [["t%d_%d" % (c, j) for j in range(25)] for c in range(k)]
    docs, labels = [], []
    for _ in range(n):
        c = rng.randrange(k)
        words = [rng.choice(topics[c]) if rng.random() < 0.3 else vocab[min(int(rng.paretovariate(1.1)) - 1, 799)]
                 for _ in range(rng.randint(3, 40))]
        docs.append(" " + " ".join(w.upper() if rng.random() < 0.1 else w for w in words) + rng.choice([".", "!", ""]))
        labels.append(c)
    return docs, np.array(labels)


def test_amazon_pipeline_in_miniature(ctx):
    import scipy.sparse as sps
    import classifier_oracle as co
    import keystone_b200 as ks
    from keystone_b200 import pipelines
    from keystone_b200.loaders import LabeledData
    docs, y = _labelled_corpus(7, 2000, 2)
    test_docs, ty = _labelled_corpus(8, 500, 2)
    conf = pipelines.AmazonReviewsConfig(commonFeatures=5000, numIters=20)
    predictor, metrics = pipelines.amazon_reviews_pipeline(ctx, LabeledData(y, docs), LabeledData(ty, test_docs), conf)
    ref_tf = to.text_features(docs, 2)
    space = to.common_sparse_features(ref_tf, 5000)
    vec = predictor.stages[5]
    assert vec.feature_space == space
    indptr, idx, val = to.vectorize(space, ref_tf)
    train_sm = vec.apply(ks.TermFrequency(lambda x: 1.0).apply(ks.NGramsFeaturizer([1, 2]).apply(
        ks.Tokenizer().apply(ks.LowerCase().apply(ks.Trim(ctx=ctx).apply(docs))))))
    _csr_equal(train_sm, (indptr, idx, val))
    A = sps.csr_matrix((val, idx, indptr), shape=(len(docs), len(space)))
    W_ref, _ = co.logistic_fit(A, y, 2, num_iters=20)
    model = predictor.stages[6]
    W = np.concatenate(model.xs, 0)[:, 1:]
    assert np.linalg.norm(W - W_ref) / np.linalg.norm(W_ref) <= 1e-9
    ti, tx, tv = to.vectorize(space, to.text_features(test_docs, 2))
    At = sps.csr_matrix((tv, tx, ti), shape=(len(test_docs), len(space)))
    pred = predictor(ctx.text(test_docs))
    Z = np.asarray(At @ W_ref).ravel()
    clear = np.abs(Z) > 1e-6 * (1.0 + np.abs(Z).max())
    assert np.array_equal(np.asarray(pred)[clear], co.logistic_predict(W_ref, At)[clear])
    ref_metrics = ks.BinaryClassifierEvaluator.evaluate(np.asarray(pred) > 0, ty > 0)
    assert (metrics.tp, metrics.fp, metrics.tn, metrics.fn) == (ref_metrics.tp, ref_metrics.fp, ref_metrics.tn, ref_metrics.fn)
    assert metrics.accuracy > 0.7


def test_newsgroups_pipeline_in_miniature(ctx):
    import scipy.sparse as sps
    import classifier_oracle as co
    from keystone_b200 import pipelines
    from keystone_b200.loaders import LabeledData
    docs, y = _labelled_corpus(9, 2000, 20)
    test_docs, ty = _labelled_corpus(10, 400, 20)
    conf = pipelines.NewsgroupsConfig(commonFeatures=5000)
    predictor, metrics = pipelines.newsgroups_pipeline(ctx, LabeledData(y, docs), LabeledData(ty, test_docs), conf)
    ref_tf = to.text_features(docs, 2)
    space = to.common_sparse_features(ref_tf, 5000)
    assert predictor.stages[5].feature_space == space
    indptr, idx, val = to.vectorize(space, ref_tf)
    A = sps.csr_matrix((val, idx, indptr), shape=(len(docs), len(space)))
    pi, theta = co.naive_bayes_fit(A, y, 20, 1.0)
    nb = predictor.stages[6]
    assert np.abs(nb.pi - pi).max() <= 1e-12 * max(1.0, np.abs(pi).max())
    assert np.abs(nb.theta - theta).max() <= 1e-12 * max(1.0, np.abs(theta).max())
    ti, tx, tv = to.vectorize(space, to.text_features(test_docs, 2))
    S = np.asarray(sps.csr_matrix((tv, tx, ti), shape=(len(test_docs), len(space))) @ theta.T) + pi
    top = np.sort(S, axis=1)
    clear = top[:, -1] - top[:, -2] > 1e-3 * (1.0 + np.abs(S).max(1))
    pred = np.asarray(predictor(ctx.text(test_docs)))
    assert np.array_equal(pred[clear], np.argmax(S, axis=1)[clear])
    assert abs(metrics.totalAccuracy - float(np.mean(pred == ty))) < 1e-12
    assert metrics.totalAccuracy > 0.5
