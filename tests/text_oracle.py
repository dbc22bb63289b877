"""Exact host restatement of the text front end (DESIGN.md section 23) for the tests: Java's String.trim / toLowerCase / split and
String.hashCode, Scala's MurmurHash3.seqHash, and the nodes of K/nodes/nlp and K/nodes/util over plain Python lists.

Terms are ``str`` (a token) or ``tuple`` of ``str`` (an n-gram).  Sparse results are CSR triples (indptr, indices, data) with the
columns of a row ascending and fp64 values.
"""
from __future__ import annotations

import math
import re
from typing import Callable, Dict, List, Sequence, Tuple

import numpy as np

_SEP = re.compile(r"[!-/:-@\[-`{-~ \t\n\x0b\f\r]+")   # \p{Punct} (32 ASCII characters) and \s of java.util.regex


def trim(s: str) -> str:
    """java.lang.String.trim: strips leading and trailing code points <= U+0020."""
    a, b = 0, len(s)
    while a < b and ord(s[a]) <= 0x20:
        a += 1
    while b > a and ord(s[b - 1]) <= 0x20:
        b -= 1
    return s[a:b]


def lower(s: str) -> str:
    """toLowerCase in the root locale, per code point by the one-to-one mapping; U+0130 -> "i" U+0307; no final-sigma rule."""
    out = []
    for ch in s:
        if ch == "\u0130":
            out.append("i\u0307")
            continue
        lo = ch.lower()
        out.append(lo if len(lo) == 1 else ch)
    return "".join(out)


def tokenize(s: str) -> List[str]:
    """String.split("[\\p{Punct}\\s]+"): a leading "" for a leading separator, trailing empty strings dropped, "" -> [""]."""
    if s == "":
        return [""]
    parts = _SEP.split(s)
    while parts and parts[-1] == "":
        parts.pop()
    return parts


def ngrams(tokens: Sequence[str], orders: Sequence[int]) -> List[tuple]:
    """NGramsFeaturizer.apply(line) (K/nodes/nlp/ngrams.scala)."""
    mn, mx = min(orders), max(orders)
    out = []
    i = 0
    while i + mn <= len(tokens):
        order = mn
        while order <= mx and i + order <= len(tokens):
            out.append(tuple(tokens[i:i + order]))
            order += 1
        i += 1
    return out


def term_frequency(terms: Sequence, fun: Callable[[float], float] = lambda x: x) -> List[tuple]:
    """TermFrequency: distinct terms in order of first occurrence, each with fun(count)."""
    counts: Dict[object, int] = {}
    for t in terms:
        counts[t] = counts.get(t, 0) + 1
    return [(t, float(fun(float(c)))) for t, c in counts.items()]


def _i32(x: int) -> int:
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >= 1 << 31 else x


def java_hash(s: str) -> int:
    """String.hashCode over UTF-16 code units."""
    b = s.encode("utf-16-be")
    h = 0
    for i in range(0, len(b), 2):
        h = (31 * h + ((b[i] << 8) | b[i + 1])) & 0xFFFFFFFF
    return _i32(h)


def _rotl(x: int, r: int) -> int:
    x &= 0xFFFFFFFF
    return ((x << r) | (x >> (32 - r))) & 0xFFFFFFFF


def _mix(h: int, data: int) -> int:
    k = (data * 0xcc9e2d51) & 0xFFFFFFFF
    k = (_rotl(k, 15) * 0x1b873593) & 0xFFFFFFFF
    h = (h ^ k) & 0xFFFFFFFF
    return (_rotl(h, 13) * 5 + 0xe6546b64) & 0xFFFFFFFF


def _finalize(h: int, length: int) -> int:
    h = (h ^ length) & 0xFFFFFFFF
    h ^= h >> 16
    h = (h * 0x85ebca6b) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xc2b2ae35) & 0xFFFFFFFF
    h ^= h >> 16
    return _i32(h)


SEQ_SEED = java_hash("Seq")


def seq_hash(words: Sequence[str]) -> int:
    """scala.util.hashing.MurmurHash3.seqHash of a Seq[String] that is not a List (orderedHash with seqSeed)."""
    h = SEQ_SEED & 0xFFFFFFFF
    for w in words:
        h = _mix(h, java_hash(w) & 0xFFFFFFFF)
    return _finalize(h, len(words))


def term_hash(t) -> int:
    """Scala's ``##``: String.hashCode for a String, seqHash for a Seq."""
    return java_hash(t) if isinstance(t, str) else seq_hash(t)


def non_negative_mod(x: int, m: int) -> int:
    r = int(math.fmod(x, m))   # Java % truncates toward zero
    return r + (m if r < 0 else 0)


def _csr(rows: List[Dict[int, float]]):
    indptr = np.zeros(len(rows) + 1, dtype=np.int64)
    idx, val = [], []
    for r, d in enumerate(rows):
        for c in sorted(d):
            idx.append(c)
            val.append(d[c])
        indptr[r + 1] = len(idx)
    return indptr, np.asarray(idx, dtype=np.int32), np.asarray(val, dtype=np.float64)


def hashing_tf(docs: Sequence[Sequence], num_features: int):
    """HashingTF(numFeatures) over documents of terms."""
    rows = []
    for terms in docs:
        d: Dict[int, float] = {}
        for t in terms:
            i = non_negative_mod(term_hash(t), num_features)
            d[i] = d.get(i, 0.0) + 1.0
        rows.append(d)
    return _csr(rows)


def ngrams_hashing_tf(docs: Sequence[Sequence[str]], orders: Sequence[int], num_features: int):
    """NGramsHashingTF(orders, numFeatures): the rolling hash of K/nodes/nlp/NGramsHashingTF.scala."""
    mn, mx = min(orders), max(orders)
    rows = []
    for line in docs:
        hashes = [java_hash(w) & 0xFFFFFFFF for w in line]
        d: Dict[int, float] = {}
        i = 0
        while i + mn <= len(line):
            h = SEQ_SEED & 0xFFFFFFFF
            for j in range(i, i + mn):
                h = _mix(h, hashes[j])
            f = non_negative_mod(_finalize(h, mn), num_features)
            d[f] = d.get(f, 0.0) + 1.0
            order = mn + 1
            while order <= mx and i + order <= len(line):
                h = _mix(h, hashes[i + order - 1])
                f = non_negative_mod(_finalize(h, order), num_features)
                d[f] = d.get(f, 0.0) + 1.0
                order += 1
            i += 1
        rows.append(d)
    return _csr(rows)


def feature_ranking(tf_docs: Sequence[Sequence[tuple]]) -> List[Tuple[object, int, int]]:
    """(term, document frequency, first flattened position), ranked by count descending, then first appearance."""
    stats: Dict[object, List[int]] = {}
    pos = 0
    for doc in tf_docs:
        for t, _ in doc:
            if t in stats:
                stats[t][0] += 1
            else:
                stats[t] = [1, pos]
            pos += 1
    ranked = sorted(stats.items(), key=lambda kv: (-kv[1][0], kv[1][1]))
    return [(t, c, f) for t, (c, f) in ranked]


def common_sparse_features(tf_docs, num_features: int) -> Dict[object, int]:
    """CommonSparseFeatures(numFeatures).fit's feature space."""
    return {t: i for i, (t, _, _) in enumerate(feature_ranking(tf_docs)[:num_features])}


def all_sparse_features(tf_docs) -> Dict[object, int]:
    return {t: i for i, (t, _, _) in enumerate(feature_ranking(tf_docs))}


def vectorize(space: Dict[object, int], tf_docs):
    """SparseFeatureVectorizer(space).apply: CSR with len(space) columns; unknown terms dropped."""
    rows = []
    for doc in tf_docs:
        d: Dict[int, float] = {}
        for t, v in doc:
            if t in space:
                d[space[t]] = d.get(space[t], 0.0) + float(v)
        rows.append(d)
    return _csr(rows)


def text_features(docs: Sequence[str], n_grams: int):
    """Trim andThen LowerCase andThen Tokenizer andThen NGramsFeaturizer(1 to n) andThen TermFrequency(x => 1)."""
    return [term_frequency(ngrams(tokenize(lower(trim(d))), range(1, n_grams + 1)), lambda x: 1.0) for d in docs]
