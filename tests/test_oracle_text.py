"""The text oracle (tests/text_oracle.py) against the literal expectations of the reference's suites (T/ = src/test/scala/keystoneml/):
T/nodes/nlp/{StringUtilsSuite,NGramSuite,HashingTFSuite,NGramsHashingTFSuite}.scala and
T/nodes/misc/{TermFrequencySuite,SparseFeatureVectorizerSuite}.scala, plus the Java / Scala hash values and split edge cases that
DESIGN.md section 23 pins.  No GPU needed."""
import math
import random

import numpy as np
import pytest

import text_oracle as to

STRINGS = ["  The quick BROWN fo.X ", " ! !.,)JumpeD. ovER the LAZy DOG.. ! "]
DATUM = "this sentence is a sentence is the some there some then there some".split(" ")


def test_string_utils_suite():
    assert [to.trim(s) for s in STRINGS] == ["The quick BROWN fo.X", "! !.,)JumpeD. ovER the LAZy DOG.. !"]
    assert [to.lower(s) for s in STRINGS] == ["  the quick brown fo.x ", " ! !.,)jumped. over the lazy dog.. ! "]
    assert [to.tokenize(s) for s in STRINGS] == [["", "The", "quick", "BROWN", "fo", "X"], ["", "JumpeD", "ovER", "the", "LAZy", "DOG"]]


def test_split_edge_cases():
    assert to.tokenize(".a.") == ["", "a"]
    assert to.tokenize("...") == []
    assert to.tokenize("") == [""]
    assert to.tokenize("a..b") == ["a", "b"]
    assert to.tokenize(to.trim("   ")) == [""]
    assert to.tokenize("x y") == ["x y"]          # a non-ASCII space is a token character
    assert to.tokenize("a\x0bb\x0cc") == ["a", "b", "c"]    # \s includes \x0B and \f


def test_lowercase_details():
    assert to.lower("İ") == "i̇"                   # as Java
    assert to.lower("Ⱥ") == "ⱥ"                    # 2 bytes -> 3 bytes
    assert len(to.lower("Ⱥ").encode()) > len("Ⱥ".encode())
    assert to.lower("ΟΔΟΣ") == "οδοσ"                        # no final-sigma rule (Java would give a final ς)
    assert to.lower("\U00010400") == "\U00010428"            # supplementary (Deseret)
    assert to.lower("ß") == "ß"


def test_ngram_suite():
    docs = [to.tokenize(s) for s in ["Pipelines are awesome", "NLP is awesome"]]
    assert [to.ngrams(d, [1]) for d in docs] == [[("Pipelines",), ("are",), ("awesome",)], [("NLP",), ("is",), ("awesome",)]]
    assert [to.ngrams(d, range(2, 4)) for d in docs] == [
        [("Pipelines", "are"), ("Pipelines", "are", "awesome"), ("are", "awesome")],
        [("NLP", "is"), ("NLP", "is", "awesome"), ("is", "awesome")]]
    assert [to.ngrams(d, [6]) for d in docs] == [[], []]


def test_hash_values():
    assert to.java_hash("hello") == 99162322
    assert to.java_hash("Seq") == 83007 == to.SEQ_SEED
    assert to.java_hash("\U0001F600") == 1772899            # the surrogate pair D83D DE00
    assert to.java_hash("") == 0
    assert to.non_negative_mod(-7, 3) == 2 and to.non_negative_mod(7, 3) == 1 and to.non_negative_mod(-6, 3) == 0
    assert to.non_negative_mod(-2 ** 31, 7) == (-(2 ** 31)) % 7


def test_hashing_tf_suite():
    datum = ["1", "2", "4", "4", "4", "4", "2"]
    indptr, idx, val = to.hashing_tf([datum], 4000)
    assert indptr[-1] == 3 and sorted(val.tolist()) == [1.0, 2.0, 4.0]
    indptr, idx, val = to.hashing_tf([datum], 2)
    assert indptr[-1] == 2 and val.sum() == len(datum)


@pytest.mark.parametrize("orders,dims", [((1, 1), 40000), ((1, 3), 40000), ((2, 3), 40000), ((1, 3), 6)])
def test_ngrams_hashing_tf_suite(orders, dims):
    r = range(orders[0], orders[1] + 1)
    a = to.hashing_tf([to.ngrams(DATUM, r)], dims)
    b = to.ngrams_hashing_tf([DATUM], r, dims)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_token_and_unigram_hashes_differ():
    a = to.hashing_tf([DATUM], 40000)
    b = to.hashing_tf([to.ngrams(DATUM, [1])], 40000)
    assert not np.array_equal(a[1], b[1])


def test_term_frequency_suite():
    assert dict(to.term_frequency(["b", "a", "c", "b", "b", "a", "b"])) == {"a": 2, "b": 4, "c": 1}
    mixed = ["b", "a", "c", ("b", "b"), ("b", "b"), 12, 12, "a", "b", 12]
    assert dict(to.term_frequency(mixed)) == {"a": 2, "b": 2, "c": 1, ("b", "b"): 2, 12: 3}
    log = dict(to.term_frequency(["b", "a", "c", "b", "b", "a", "b"], lambda x: math.log(x + 1)))
    assert log == {"a": math.log(3), "b": math.log(5), "c": math.log(2)}
    assert [t for t, _ in to.term_frequency(["b", "a", "c", "b"])] == ["b", "a", "c"]   # order of first occurrence


def test_sparse_feature_vectorizer_suite():
    space = {"First": 0, "Second": 1, "Third": 2}
    indptr, idx, val = to.vectorize(space, [[("Third", 4.0), ("Fourth", 6.0), ("First", 1.0)]])
    assert idx.tolist() == [0, 2] and val.tolist() == [1.0, 4.0]
    train = [[("First", 0.0), ("Second", 6.0)], [("Third", 3.0), ("Second", 4.0)]]
    space = to.all_sparse_features(train)
    assert space == {"Second": 0, "First": 1, "Third": 2}
    _, idx, val = to.vectorize(space, [[("Third", 4.0), ("Fourth", 6.0), ("First", 1.0)]])
    dense = np.zeros(3)
    dense[idx] = val
    assert sorted(dense.tolist()) == [0.0, 1.0, 4.0] and dense[space["First"]] == 1.0 and dense[space["Third"]] == 4.0
    train = [[("First", 0.0), ("Second", 6.0)], [("Third", 3.0), ("Second", 4.8)], [("Third", 7.0), ("Fourth", 5.0)],
             [("Fifth", 5.0), ("Second", 7.3)]]
    space = to.common_sparse_features(train, 2)
    assert space == {"Second": 0, "Third": 1}
    _, idx, val = to.vectorize(space, [[("Third", 4.0), ("Seventh", 8.0), ("Second", 1.3), ("Fourth", 6.0), ("First", 1.0)]])
    assert val.tolist() == [1.3, 4.0]


def test_all_sparse_features_order_is_first_appearance_when_counts_tie():
    train = [[("b", 1.0), ("a", 1.0)], [("c", 1.0)]]
    assert to.all_sparse_features(train) == {"b": 0, "a": 1, "c": 2}


def test_selection_keeps_the_largest_counts():
    rng = random.Random(3)
    vocab = [f"w{i}" for i in range(60)]
    for trial in range(20):
        docs = []
        for _ in range(rng.randint(1, 40)):
            toks = [rng.choice(vocab[:rng.randint(1, 60)]) for _ in range(rng.randint(0, 12))]
            docs.append(to.term_frequency(toks, lambda x: 1.0))
        ranking = to.feature_ranking(docs)
        k = rng.randint(1, max(1, len(ranking)))
        chosen = to.common_sparse_features(docs, k)
        counts = {t: c for t, c, _ in ranking}
        sel = [counts[t] for t in chosen]
        rest = [c for t, c in counts.items() if t not in chosen]
        assert not rest or min(sel) >= max(rest)
        assert list(chosen.values()) == list(range(len(chosen)))


def test_pipeline_features_in_miniature():
    docs = ["  Great product!! ", "great, GREAT product", ""]
    tf = to.text_features(docs, 2)
    assert tf[0] == [(("great",), 1.0), (("great", "product"), 1.0), (("product",), 1.0)]
    assert tf[1] == [(("great",), 1.0), (("great", "great"), 1.0), (("great", "product"), 1.0), (("product",), 1.0)]
    assert tf[2] == [(("",), 1.0)]
