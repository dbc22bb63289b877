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
