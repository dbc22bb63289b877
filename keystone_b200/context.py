"""GPU context and row-sharded device datasets (host side of the C ABI).

``Context`` = one process / one GPU (``ks_ctx_create``).  ``DeviceMatrix`` is this rank's shard of
a row-partitioned dataset -- the stand-in for the reference's ``RDD[DenseVector[Double]]`` at the
estimator boundary (SURVEY.md 8a/a11).  ``LazyFeatures`` is the un-materialised output of gathered
CosineRandomFeatures nodes: the fit regenerates every feature block from ``x_in`` instead of storing
N x D (the reference relies on Spark's lazy RDDs for the same thing, K/workflow/Pipeline.scala:81-96).
"""
from __future__ import annotations

import ctypes as C
import json
from typing import List, Optional, Sequence

import numpy as np

from . import _capi
from ._capi import KeystoneError, check, lib


def shard_range(n_rows: int, rank: int, world: int):
    """Contiguous, near-equal row ranges; the first ``n % world`` ranks take one extra row
    (SURVEY.md 8e: rows shard naturally; every per-partition quantity in the reference is a row sum)."""
    base, rem = divmod(int(n_rows), int(world))
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


class Context:
    def __init__(self, device: int = 0, rank: int = 0, world_size: int = 1, nccl_id: Optional[bytes] = None):
        self.handle = 0
        self.rank, self.world_size, self.device = rank, world_size, device
        h = C.c_int64(0)
        idbuf = None
        if nccl_id is not None:
            idbuf = (C.c_uint8 * _capi.KS_NCCL_ID_BYTES).from_buffer_copy(nccl_id)
        rc = lib().ks_ctx_create(device, rank, world_size, idbuf, C.byref(h))
        if rc != 0:
            check(0, rc)
        self.handle = h.value

    # ---- distributed bring-up over an existing torch.distributed group (plumbing only) ----
    @staticmethod
    def new_nccl_id() -> bytes:
        buf = (C.c_uint8 * _capi.KS_NCCL_ID_BYTES)()
        rc = lib().ks_nccl_unique_id(buf)
        if rc != 0:
            check(0, rc)
        return bytes(buf)

    @classmethod
    def from_torch_distributed(cls, device: Optional[int] = None) -> "Context":
        import os
        import torch.distributed as dist

        rank, world = dist.get_rank(), dist.get_world_size()
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", rank))
        ids = [cls.new_nccl_id() if rank == 0 else None]
        if world > 1:
            dist.broadcast_object_list(ids, src=0)
        return cls(device=device, rank=rank, world_size=world, nccl_id=ids[0] if world > 1 else None)

    def close(self) -> None:
        if self.handle:
            lib().ks_ctx_destroy(self.handle)
            self.handle = 0

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, name: str, value: int) -> None:
        check(self.handle, lib().ks_ctx_set_option(self.handle, name.encode(), int(value)))

    def synchronize(self) -> None:
        check(self.handle, lib().ks_ctx_synchronize(self.handle))

    def launch_count(self) -> int:
        v = C.c_int64(0)
        check(self.handle, lib().ks_ctx_launch_count(self.handle, C.byref(v)))
        return v.value

    def last_fit_stats(self) -> dict:
        n = C.c_int64(0)   # the JSON grows with the fit (DenseLBFGSwithL2 reports its loss history): size the buffer from it
        check(self.handle, lib().ks_last_fit_stats_json_size(self.handle, C.byref(n)))
        buf = C.create_string_buffer(max(int(n.value), 1))
        check(self.handle, lib().ks_last_fit_stats_json(self.handle, buf, len(buf)))
        s = buf.value.decode()
        return json.loads(s) if s else {}

    # ---- dataset constructors ----
    def matrix(self, arr: np.ndarray) -> "DeviceMatrix":
        arr = np.asarray(arr)
        if arr.ndim == 1:
            arr = arr[None, :]
        if arr.dtype == np.float32:
            a = np.ascontiguousarray(arr)
            fn = lib().ks_matrix_from_host_f32
        else:
            a = np.ascontiguousarray(arr, dtype=np.float64)
            fn = lib().ks_matrix_from_host_f64
        h = C.c_int64(0)
        check(self.handle, fn(self.handle, a.ctypes.data_as(C.c_void_p), a.shape[0], a.shape[1], a.shape[1], C.byref(h)))
        return DeviceMatrix(self, h.value, a.shape[0], a.shape[1])

    def matrix_from_partitions(self, parts: Sequence[np.ndarray]) -> "DeviceMatrix":
        """One device matrix from several host row chunks (an executor's RDD partitions), uploaded chunk by chunk."""
        parts = [np.atleast_2d(np.asarray(p)) for p in parts]
        rows, cols = sum(p.shape[0] for p in parts), parts[0].shape[1]
        h = C.c_int64(0)
        check(self.handle, lib().ks_matrix_create(self.handle, rows, cols, C.byref(h)))
        out = DeviceMatrix(self, h.value, rows, cols)
        r0 = 0
        for p in parts:
            if p.dtype == np.float32:
                a, fn = np.ascontiguousarray(p), lib().ks_matrix_write_rows_f32
            else:
                a, fn = np.ascontiguousarray(p, dtype=np.float64), lib().ks_matrix_write_rows_f64
            check(self.handle, fn(self.handle, h.value, r0, a.ctypes.data_as(C.c_void_p), a.shape[0], a.shape[1]))
            r0 += a.shape[0]
        return out

    def synthetic_normal(self, n_rows: int, n_cols: int, seed: int, global_row_offset: int = 0, mean: float = 0.0,
                         stddev: float = 1.0) -> "DeviceMatrix":
        h = C.c_int64(0)
        check(self.handle, lib().ks_matrix_synthetic_normal(self.handle, n_rows, n_cols, seed, global_row_offset, mean, stddev,
                                                             C.byref(h)))
        return DeviceMatrix(self, h.value, n_rows, n_cols)

    def sparse(self, obj) -> "SparseMatrix":
        """This rank's rows of a sparse matrix, uploaded as CSR (``ks_sparse_from_host_csr``).  ``obj`` is anything with ``indptr``,
        ``indices``, ``data`` and ``shape`` (a scipy CSR matrix qualifies; scipy is not needed), or a tuple
        ``(indptr, indices, data, n_cols)``.  Repeated (row, column) entries add up; unsorted indices and empty rows are legal."""
        if isinstance(obj, tuple):
            if len(obj) != 4:
                raise KeystoneError(-1, "a sparse tuple is (indptr, indices, data, n_cols)")
            indptr, indices, data, n_cols = obj
            n_rows = len(indptr) - 1
        else:
            indptr, indices, data = obj.indptr, obj.indices, obj.data
            n_rows, n_cols = int(obj.shape[0]), int(obj.shape[1])
        indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        indices = np.asarray(indices)
        data = np.ascontiguousarray(data, dtype=np.float64)
        n_cols = int(n_cols)
        if indptr.ndim != 1 or indptr.shape[0] != n_rows + 1 or n_rows < 0:
            raise KeystoneError(-1, "indptr must hold n_rows + 1 offsets")
        nnz = int(indptr[-1])
        if indices.shape != (nnz,) or data.shape != (nnz,):
            raise KeystoneError(-1, f"indptr[n_rows] = {nnz} does not match {indices.shape[0]} indices and {data.shape[0]} values")
        if nnz and (int(indices.min()) < 0 or int(indices.max()) >= n_cols):   # before the int32 cast, which would wrap them
            raise KeystoneError(-1, "a column index lies outside [0, n_cols)")
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        h = C.c_int64(0)
        check(self.handle, lib().ks_sparse_from_host_csr(self.handle, indptr.ctypes.data_as(C.c_void_p), indices.ctypes.data_as(C.c_void_p),
                                                          data.ctypes.data_as(C.c_void_p), n_rows, n_cols, C.byref(h)))
        return SparseMatrix(self, h.value, n_rows, n_cols, nnz)

    def text(self, docs: Sequence) -> "TextBatch":
        """A batch of documents on the device (``ks_text_from_host``): each ``str`` is encoded as UTF-8 (a lone surrogate is
        rejected here); ``bytes`` items are taken as they are, and invalid UTF-8 among them is found on the device and rejected."""
        data, off = _encode_all(docs, "document")
        h = C.c_int64(0)
        check(self.handle, lib().ks_text_from_host(self.handle, data.ctypes.data_as(C.c_void_p), data.shape[0], off.ctypes.data_as(C.c_void_p),
                                                    off.shape[0] - 1, C.byref(h)))
        return TextBatch(self, h.value, off.shape[0] - 1)

    def tokens(self, docs: Sequence[Sequence[str]]) -> "TokenBatch":
        """A token batch from host lists of strings, one list per document (``ks_tokens_from_host``)."""
        flat = [t for d in docs for t in d]
        data, toff = _encode_all(flat, "token")
        doff = np.zeros(len(docs) + 1, dtype=np.int64)
        doff[1:] = np.cumsum([len(d) for d in docs])
        h = C.c_int64(0)
        check(self.handle, lib().ks_tokens_from_host(self.handle, data.ctypes.data_as(C.c_void_p), data.shape[0], toff.ctypes.data_as(C.c_void_p),
                                                      len(flat), doff.ctypes.data_as(C.c_void_p), len(docs), C.byref(h)))
        return TokenBatch(self, h.value, len(docs))

    def term_frequencies(self, docs: Sequence[Sequence[tuple]]) -> "TermFrequencyBatch":
        """A term-frequency batch from host lists of ``(term, value)`` pairs, one list per document: a term is a ``str`` or a tuple
        of one to four ``str`` (``ks_tf_from_host``)."""
        terms = [t for d in docs for t, _ in d]
        tokens, first, order = _flatten_terms(terms)
        values = np.ascontiguousarray([float(v) for d in docs for _, v in d], dtype=np.float64)
        doff = np.zeros(len(docs) + 1, dtype=np.int64)
        doff[1:] = np.cumsum([len(d) for d in docs])
        tk = self.tokens([tokens])
        h = C.c_int64(0)
        check(self.handle, lib().ks_tf_from_host(self.handle, tk.handle, first.ctypes.data_as(C.c_void_p), order.ctypes.data_as(C.c_void_p),
                                                  values.ctypes.data_as(C.c_void_p), len(terms), doff.ctypes.data_as(C.c_void_p), len(docs),
                                                  C.byref(h)))
        return TermFrequencyBatch(self, h.value, len(docs), tk)

    def labels_from_classes(self, classes: np.ndarray, num_classes: int) -> "DeviceMatrix":
        cls = np.ascontiguousarray(classes, dtype=np.int32)
        h = C.c_int64(0)
        check(self.handle, lib().ks_labels_from_classes(self.handle, cls.ctypes.data_as(C.c_void_p), cls.shape[0], num_classes,
                                                         C.byref(h)))
        return DeviceMatrix(self, h.value, cls.shape[0], num_classes)


class Dataset:
    """Marker base: something a Transformer / Estimator accepts as a batch."""


class DeviceMatrix(Dataset):
    def __init__(self, ctx: Context, handle: int, rows: int, cols: int):
        self.ctx, self.handle, self.rows, self.cols = ctx, handle, rows, cols

    @property
    def shape(self):
        return (self.rows, self.cols)

    def to_numpy(self, dtype=np.float64) -> np.ndarray:
        out = np.empty((self.rows, self.cols), dtype=dtype)
        if self.rows == 0:
            return out
        fn = lib().ks_matrix_to_host_f64 if dtype == np.float64 else lib().ks_matrix_to_host_f32
        check(self.ctx.handle, fn(self.ctx.handle, self.handle, out.ctypes.data_as(C.c_void_p), self.cols))
        return out

    def free(self) -> None:
        if self.handle and self.ctx.handle:
            lib().ks_matrix_destroy(self.ctx.handle, self.handle)
        self.handle = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class SparseMatrix(Dataset):
    """This rank's rows of a row-sharded sparse matrix on the device (CSR plus a CSC copy): the stand-in for the reference's
    ``RDD[SparseVector[Double]]``.  Only the sparse nodes take it; the dense nodes reject it."""

    def __init__(self, ctx: Context, handle: int, rows: int, cols: int, nnz: int):
        self.ctx, self.handle, self.rows, self.cols, self.nnz = ctx, handle, rows, cols, nnz

    @property
    def shape(self):
        return (self.rows, self.cols)

    def to_csr(self):
        """(indptr int64, indices int32, data fp64) of this rank's rows as stored on the device."""
        indptr = np.empty(self.rows + 1, dtype=np.int64)
        indices = np.empty(self.nnz, dtype=np.int32)
        data = np.empty(self.nnz, dtype=np.float64)
        check(self.ctx.handle, lib().ks_sparse_to_host_csr(self.ctx.handle, self.handle, indptr.ctypes.data_as(C.c_void_p),
                                                            indices.ctypes.data_as(C.c_void_p), data.ctypes.data_as(C.c_void_p)))
        return indptr, indices, data

    def free(self) -> None:
        if self.handle and self.ctx.handle:
            lib().ks_sparse_destroy(self.ctx.handle, self.handle)
        self.handle = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class LazyFeatures(Dataset):
    """cos(X W_i^T + b_i) for a list of CosineRandomFeatures handles, concatenated (VectorCombiner)."""

    def __init__(self, x_in: DeviceMatrix, rf_handles: Sequence[int], n_out: Sequence[int], owners: Sequence[object]):
        self.ctx = x_in.ctx
        self.x_in = x_in
        self.rf_handles = list(rf_handles)
        self.n_out = list(n_out)
        self.owners = list(owners)  # keep the node objects (and their device parameters) alive

    @property
    def rows(self):
        return self.x_in.rows

    @property
    def cols(self):
        return int(sum(self.n_out))

    @property
    def shape(self):
        return (self.rows, self.cols)

    def concat(self, other: "LazyFeatures") -> "LazyFeatures":
        if other.x_in is not self.x_in:
            raise KeystoneError(-1, "gathered CosineRandomFeatures branches must share the same input")
        return LazyFeatures(self.x_in, self.rf_handles + other.rf_handles, self.n_out + other.n_out, self.owners + other.owners)

    def materialize(self) -> DeviceMatrix:
        parts: List[np.ndarray] = []
        if len(self.rf_handles) == 1:
            h = C.c_int64(0)
            check(self.ctx.handle, lib().ks_cosine_rf_apply(self.ctx.handle, self.rf_handles[0], self.x_in.handle, C.byref(h)))
            return DeviceMatrix(self.ctx, h.value, self.rows, self.n_out[0])
        for rf, n in zip(self.rf_handles, self.n_out):
            h = C.c_int64(0)
            check(self.ctx.handle, lib().ks_cosine_rf_apply(self.ctx.handle, rf, self.x_in.handle, C.byref(h)))
            parts.append(DeviceMatrix(self.ctx, h.value, self.rows, n).to_numpy(np.float32))
        return self.ctx.matrix(np.concatenate(parts, axis=1))

    def to_numpy(self, dtype=np.float64) -> np.ndarray:
        return self.materialize().to_numpy(dtype)


def feature_source_args(data: Dataset):
    """(features_handle, x_in_handle, rfs_array, n_rfs) for the C ABI's feature-source parameters."""
    if isinstance(data, DeviceMatrix):
        return data.handle, 0, None, 0
    if isinstance(data, LazyFeatures):
        arr = (C.c_int64 * len(data.rf_handles))(*data.rf_handles)
        return 0, data.x_in.handle, arr, len(data.rf_handles)
    raise KeystoneError(-1, f"unsupported dataset type {type(data).__name__}")


# ---- text batches (text.cu, DESIGN.md section 23) ----
def _encode_all(items: Sequence, what: str):
    """(uint8 bytes, int64 offsets) of the UTF-8 encodings of ``items`` (``str`` or ``bytes``)."""
    parts = []
    for i, x in enumerate(items):
        if isinstance(x, (bytes, bytearray)):
            parts.append(bytes(x))
        elif isinstance(x, str):
            try:
                parts.append(x.encode("utf-8"))
            except UnicodeEncodeError as e:
                raise KeystoneError(-1, f"{what} {i} holds a lone surrogate (U+{ord(x[e.start]):04X}), which has no UTF-8 form") from None
        else:
            raise KeystoneError(-1, f"{what} {i} is a {type(x).__name__}, not a str")
    off = np.zeros(len(parts) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(p) for p in parts])
    data = np.frombuffer(b"".join(parts), dtype=np.uint8) if parts else np.zeros(0, dtype=np.uint8)
    return np.ascontiguousarray(data), off


def _flatten_terms(terms: Sequence):
    """Terms (``str``, or tuples of one to four ``str``) as (tokens, first token, order): order 0 marks a ``str``."""
    tokens: List[str] = []
    first = np.zeros(len(terms), dtype=np.int64)
    order = np.zeros(len(terms), dtype=np.int32)
    for i, t in enumerate(terms):
        first[i] = len(tokens)
        if isinstance(t, str):
            tokens.append(t)
        elif isinstance(t, tuple) and 1 <= len(t) <= 4 and all(isinstance(w, str) for w in t):
            tokens.extend(t)
            order[i] = len(t)
        else:
            raise KeystoneError(-1, f"term {t!r}: a term on the device is a str or a tuple of one to four str")
    return tokens, first, order


def _text_array(ctx: Context, handle: int, which: int, dtype) -> np.ndarray:
    n = C.c_int64(0)
    check(ctx.handle, lib().ks_text_array_size(ctx.handle, handle, which, C.byref(n)))
    out = np.empty(n.value, dtype=dtype)
    check(ctx.handle, lib().ks_text_array(ctx.handle, handle, which, out.ctypes.data_as(C.c_void_p), n.value))
    return out


def _host_tokens(ctx: Context, handle: int) -> List[str]:
    data = _text_array(ctx, handle, _capi.KS_TEXT_BYTES, np.uint8).tobytes()
    tb = _text_array(ctx, handle, _capi.KS_TEXT_TOKEN_BEGIN, np.int64)
    te = _text_array(ctx, handle, _capi.KS_TEXT_TOKEN_END, np.int64)
    return [data[a:b].decode("utf-8") for a, b in zip(tb.tolist(), te.tolist())]


def _host_terms(ctx: Context, handle: int) -> list:
    toks = _host_tokens(ctx, handle)
    first = _text_array(ctx, handle, _capi.KS_TEXT_TERM_FIRST, np.int64).tolist()
    order = _text_array(ctx, handle, _capi.KS_TEXT_TERM_ORDER, np.int32).tolist()
    return [toks[f] if o == 0 else tuple(toks[f:f + o]) for f, o in zip(first, order)]


class _TextObject(Dataset):
    def __init__(self, ctx: Context, handle: int, n_docs: int):
        self.ctx, self.handle, self.n_docs = ctx, handle, n_docs

    def __len__(self):
        return self.n_docs

    def free(self) -> None:
        if self.handle and self.ctx.handle:
            lib().ks_text_destroy(self.ctx.handle, self.handle)
        self.handle = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class TextBatch(_TextObject):
    """This rank's documents on the device: UTF-8 bytes and int64 document offsets (the reference's ``RDD[String]``)."""

    def to_host(self) -> List[str]:
        data = _text_array(self.ctx, self.handle, _capi.KS_TEXT_BYTES, np.uint8).tobytes()
        off = _text_array(self.ctx, self.handle, _capi.KS_TEXT_DOC_OFFSETS, np.int64).tolist()
        return [data[off[d]:off[d + 1]].decode("utf-8") for d in range(self.n_docs)]


class TokenBatch(_TextObject):
    """The tokens of each document (``RDD[Seq[String]]``): byte ranges into the text they came from, with Java's
    ``String.hashCode`` and a content hash of each."""

    def to_host(self) -> List[List[str]]:
        toks = _host_tokens(self.ctx, self.handle)
        off = _text_array(self.ctx, self.handle, _capi.KS_TEXT_DOC_OFFSETS, np.int64).tolist()
        return [toks[off[d]:off[d + 1]] for d in range(self.n_docs)]

    def java_hashes(self) -> np.ndarray:
        """``String.hashCode`` of every token, in order (int32)."""
        return _text_array(self.ctx, self.handle, _capi.KS_TEXT_TOKEN_JAVA_HASH, np.int32)


class NGramBatch(Dataset):
    """The n-grams of the given orders of a token batch (``RDD[Seq[Seq[String]]]``), lazy: the device emits them inside the node
    that consumes them.  Per document they come in ``NGramsFeaturizer``'s order: for each position, each order ascending."""

    def __init__(self, tokens: TokenBatch, min_order: int, max_order: int):
        self.ctx, self.tokens, self.min_order, self.max_order = tokens.ctx, tokens, int(min_order), int(max_order)
        self.n_docs = tokens.n_docs

    def __len__(self):
        return self.n_docs

    def to_host(self) -> List[List[tuple]]:
        out = []
        for toks in self.tokens.to_host():
            grams = []
            for i in range(len(toks) - self.min_order + 1):
                for o in range(self.min_order, self.max_order + 1):
                    if i + o > len(toks):
                        break
                    grams.append(tuple(toks[i:i + o]))
            out.append(grams)
        return out


class TermFrequencyBatch(_TextObject):
    """Per document its distinct terms with a value (``RDD[Seq[(T, Double)]]``); ``max_count`` is the largest count in the batch
    (0 for an uploaded batch, which carries values only)."""

    def __init__(self, ctx: Context, handle: int, n_docs: int, tokens: Dataset, max_count: int = 0):
        super().__init__(ctx, handle, n_docs)
        self.tokens, self.max_count = tokens, int(max_count)

    def to_host(self) -> List[List[tuple]]:
        terms = _host_terms(self.ctx, self.handle)
        values = _text_array(self.ctx, self.handle, _capi.KS_TEXT_TERM_VALUE, np.float64).tolist()
        off = _text_array(self.ctx, self.handle, _capi.KS_TEXT_DOC_OFFSETS, np.int64).tolist()
        return [list(zip(terms[off[d]:off[d + 1]], values[off[d]:off[d + 1]])) for d in range(self.n_docs)]
