"""Node library of the hot path: same class names, constructor arguments and semantics as the
reference nodes; the bodies marshal to the C ABI (which launches the sm_90a kernels).

Reference classes (K/ = src/main/scala/keystoneml/):
  CosineRandomFeatures                K/nodes/stats/CosineRandomFeatures.scala:19-60
  StandardScaler / StandardScalerModel K/nodes/stats/StandardScaler.scala:16-59
  VectorSplitter                      K/nodes/util/VectorSplitter.scala:10-36
  VectorCombiner                      K/nodes/util/VectorCombiner.scala:11-14
  ClassLabelIndicatorsFromIntLabels   K/nodes/util/ClassLabelIndicators.scala:15-29
  MaxClassifier                       K/nodes/util/MaxClassifier.scala:9-11
  BlockLeastSquaresEstimator          K/nodes/learning/BlockLinearMapper.scala:199-283
  BlockWeightedLeastSquaresEstimator  K/nodes/learning/BlockWeightedLeastSquares.scala:36-84
  BlockLinearMapper                   K/nodes/learning/BlockLinearMapper.scala:22-138
  LinearMapper / LinearMapEstimator   K/nodes/learning/LinearMapper.scala:18-116
  DenseLBFGSwithL2                    K/nodes/learning/LBFGS.scala:135-192
  LeastSquaresDenseGradient           K/nodes/learning/Gradient.scala:29-53

Batches are ``DeviceMatrix`` / ``LazyFeatures`` (this rank's rows); 2-D numpy arrays are uploaded on
the fly when a ``Context`` was given to the node.  No node computes on the host.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional, Sequence

import numpy as np

from . import _capi
from ._capi import KeystoneError, check, lib
from .context import Context, Dataset, DeviceMatrix, LazyFeatures, feature_source_args
from .workflow import Estimator, LabelEstimator, Transformer, WeightedNode


def _as_dataset(ctx: Optional[Context], data) -> Dataset:
    if isinstance(data, Dataset):
        return data
    if ctx is None:
        raise KeystoneError(-1, "numpy input needs a Context (pass ctx= to the node)")
    return ctx.matrix(np.asarray(data))


# ------------------------------------------------------------------------------------------
class CosineRandomFeatures(Transformer):
    """cos(x W^T + b); W is (numOutputFeatures x numInputFeatures), b has numOutputFeatures entries."""

    def __init__(self, ctx: Context, W: np.ndarray, b: np.ndarray):
        W = np.asarray(W, dtype=np.float64)
        b = np.asarray(b, dtype=np.float64)
        if b.shape[0] != W.shape[0]:  # CosineRandomFeatures.scala:24
            raise ValueError("# of rows in W and size of b should match")
        self.ctx, self.n_out, self.n_in = ctx, W.shape[0], W.shape[1]
        wcol = np.asfortranarray(W)  # Breeze DenseMatrix storage
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_cosine_rf_create(ctx.handle, wcol.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
                                                     self.n_out, self.n_in, C.byref(h)))
        self.handle = h.value

    @classmethod
    def create(cls, ctx: Context, num_input_features: int, num_output_features: int, gamma: float,
               rng: Optional[np.random.Generator] = None, w_dist: str = "gaussian") -> "CosineRandomFeatures":
        """Companion-object factory (CosineRandomFeatures.scala:51-60): W = gamma * rand(wDist), b = 2 pi U[0,1)."""
        rng = rng or np.random.default_rng()
        if w_dist == "gaussian":
            W = rng.standard_normal((num_output_features, num_input_features))
        elif w_dist == "cauchy":
            W = rng.standard_cauchy((num_output_features, num_input_features))
        else:
            raise ValueError(w_dist)
        return cls(ctx, W * gamma, rng.random(num_output_features) * (2 * math.pi))

    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 1
        ds = _as_dataset(self.ctx, data)
        if not isinstance(ds, DeviceMatrix):
            raise KeystoneError(-1, "CosineRandomFeatures expects a dense input batch")
        out = LazyFeatures(ds, [self.handle], [self.n_out], [self])
        return out.to_numpy()[0] if single else out

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                lib().ks_cosine_rf_destroy(self.ctx.handle, self.handle)
        except Exception:
            pass


class _FeatureMapHandle:
    """Owns a dense feature-map handle of the library (PaddedFFT / rectified maps; same handle space as CosineRandomFeatures)."""

    def __init__(self, ctx: Context, handle: int):
        self.ctx, self.handle = ctx, handle

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                lib().ks_cosine_rf_destroy(self.ctx.handle, self.handle)
        except Exception:
            pass


class _SignedInput(Dataset):
    """Lazy ``x .* signs`` (RandomSignNode output): fused into the PaddedFFT map that consumes it."""

    def __init__(self, x: DeviceMatrix, signs: np.ndarray):
        self.ctx, self.x, self.signs = x.ctx, x, signs
        self.rows, self.cols = x.rows, x.cols

    def materialize(self) -> DeviceMatrix:
        h = C.c_int64(0)
        check(self.ctx.handle, lib().ks_matrix_map(self.ctx.handle, self.x.handle, 0, self.signs.ctypes.data_as(C.c_void_p), 0.0, 0.0,
                                                    C.byref(h)))
        return DeviceMatrix(self.ctx, h.value, self.rows, self.cols)

    def to_numpy(self, dtype=np.float64) -> np.ndarray:
        return self.materialize().to_numpy(dtype)


class _FFTFeatures(LazyFeatures):
    """Lazy PaddedFFT output (optionally of a sign-flipped input): a LazyFeatures whose single map is the FFT cosine matrix;
    a following LinearRectifier swaps the map for the rectified one."""

    def __init__(self, x: DeviceMatrix, signs: Optional[np.ndarray], rectifier=None):
        ctx = x.ctx
        self.signs, self.rectifier = signs, rectifier
        h = C.c_int64(0)
        sp = None if signs is None else signs.ctypes.data_as(C.c_void_p)
        rect, mx, al = (0, 0.0, 0.0) if rectifier is None else (1, float(rectifier[0]), float(rectifier[1]))
        check(ctx.handle, lib().ks_padded_fft_create(ctx.handle, sp, x.cols, rect, mx, al, C.byref(h)))
        owner = _FeatureMapHandle(ctx, h.value)
        n_out = PaddedFFT.next_positive_power_of_two(x.cols) // 2
        super().__init__(x, [h.value], [n_out], [owner])


class RandomSignNode(Transformer):
    """``in :* signs`` (K/nodes/stats/RandomSignNode.scala:11-16).  On a device batch the product is lazy and folds into the
    PaddedFFT map that follows."""

    def __init__(self, signs: np.ndarray, ctx: Optional[Context] = None):
        self.signs = np.ascontiguousarray(signs, dtype=np.float64)
        self.ctx = ctx

    @classmethod
    def create(cls, size: int, rng: Optional[np.random.Generator] = None, ctx: Optional[Context] = None) -> "RandomSignNode":
        """Companion factory (:19-23): 2 * Binomial(1, 0.5) - 1 per element."""
        rng = rng or np.random.default_rng()
        return cls(2.0 * rng.integers(0, 2, size).astype(np.float64) - 1.0, ctx)

    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 1
        ds = _as_dataset(self.ctx, data)
        if not isinstance(ds, DeviceMatrix):
            ds = ds.materialize()
        if ds.cols != self.signs.shape[0]:
            raise ValueError("signs and input have different lengths")
        out = _SignedInput(ds, self.signs)
        return out.to_numpy()[0] if single else out


class PaddedFFT(Transformer):
    """Pads to the next power of two P and returns the real part of the first P / 2 FFT bins
    (K/nodes/stats/PaddedFFT.scala:13-21) -- on the device a fixed cosine-matrix product on the tensor cores."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    @staticmethod
    def next_positive_power_of_two(i: int) -> int:
        return 1 << max(0, (int(i) - 1).bit_length())

    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 1
        if isinstance(data, _SignedInput):
            out = _FFTFeatures(data.x, data.signs)
        else:
            ds = _as_dataset(self.ctx, data)
            if not isinstance(ds, DeviceMatrix):
                ds = ds.materialize()
            out = _FFTFeatures(ds, None)
        return out.to_numpy()[0] if single else out


class LinearRectifier(Transformer):
    """``max(maxVal, x - alpha)`` (K/nodes/stats/LinearRectifier.scala:12-17); after PaddedFFT it becomes the epilogue of the
    FFT GEMM."""

    def __init__(self, max_val: float = 0.0, alpha: float = 0.0, ctx: Optional[Context] = None):
        self.max_val, self.alpha, self.ctx = float(max_val), float(alpha), ctx

    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 1
        if isinstance(data, _FFTFeatures) and data.rectifier is None:
            return _FFTFeatures(data.x_in, data.signs, (self.max_val, self.alpha))
        ds = _as_dataset(self.ctx, data)
        if not isinstance(ds, DeviceMatrix):
            ds = ds.materialize()
        h = C.c_int64(0)
        check(ds.ctx.handle, lib().ks_matrix_map(ds.ctx.handle, ds.handle, 1, None, self.max_val, self.alpha, C.byref(h)))
        out = DeviceMatrix(ds.ctx, h.value, ds.rows, ds.cols)
        return out.to_numpy()[0] if single else out


class _ConvHandle:
    def __init__(self, ctx: Context, handle: int):
        self.ctx, self.handle = ctx, handle

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                lib().ks_convolver_destroy(self.ctx.handle, self.handle)
        except Exception:
            pass


class _ConvolvedImages(Dataset):
    """Lazy output of Convolver [-> SymmetricRectifier [-> Pooler]] on an image batch: the chain runs as ONE fused launch per image
    chunk when it is materialised (``ImageVectorizer`` / ``to_numpy``)."""

    def __init__(self, images: DeviceMatrix, conv: "Convolver", rect=None, pool=None):
        self.ctx, self.images, self.conv, self.rect, self.pool = images.ctx, images, conv, rect, pool
        self.rows = images.rows

    def materialize(self) -> DeviceMatrix:
        if self.rect is not None and self.pool is None:
            raise KeystoneError(-1, "SymmetricRectifier on convolved images is fused with the Pooler that follows it: chain a Pooler")
        stride, size = self.pool if self.pool else (0, 0)
        max_val, alpha = self.rect if self.rect else (0.0, 0.0)
        if self.pool and self.rect is None:
            raise KeystoneError(-1, "Pooler after Convolver needs the SymmetricRectifier in between (the fused kernel's epilogue)")
        h = C.c_int64(0)
        check(self.ctx.handle, lib().ks_convolver_apply(self.ctx.handle, self.conv._h.handle, self.images.handle, stride, size,
                                                         float(max_val), float(alpha), C.byref(h)))
        rows, cols = C.c_int64(0), C.c_int64(0)
        check(self.ctx.handle, lib().ks_matrix_shape(self.ctx.handle, h.value, C.byref(rows), C.byref(cols)))
        return DeviceMatrix(self.ctx, h.value, rows.value, cols.value)

    def to_numpy(self, dtype=np.float64) -> np.ndarray:
        return self.materialize().to_numpy(dtype)


class Convolver(Transformer):
    """``new Convolver(filters, imgWidth, imgHeight, imgChannels, whitener, normalizePatches, varConstant)``
    (K/nodes/images/Convolver.scala:20-47).  filters: (numFilters x convSize^2*channels), columns in packFilters order, already
    whitened when a whitener is used; ``whitener_means`` = the whitener's means (the only part of the ZCAWhitener that apply uses,
    :196-199).  Image batches are device matrices whose rows are images in ImageVectorizer order."""

    def __init__(self, ctx: Context, filters: np.ndarray, img_width: int, img_height: int, img_channels: int,
                 whitener_means: Optional[np.ndarray] = None, normalize_patches: bool = True, var_constant: float = 10.0):
        filters = np.asarray(filters, dtype=np.float64)
        self.ctx, self.n_filters = ctx, filters.shape[0]
        self.x_dim, self.y_dim, self.ch = img_width, img_height, img_channels
        self.conv_size = int(round(math.sqrt(filters.shape[1] / img_channels)))          # Convolver.scala:30
        if self.conv_size * self.conv_size * img_channels != filters.shape[1]:
            raise ValueError("filters must be square patches of the image's channel count")
        fcol = np.asfortranarray(filters)
        wm = None if whitener_means is None else np.ascontiguousarray(whitener_means, dtype=np.float64)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_convolver_create(ctx.handle, fcol.ctypes.data_as(C.c_void_p), self.n_filters, img_width, img_height,
                                                     img_channels, self.conv_size, None if wm is None else wm.ctypes.data_as(C.c_void_p),
                                                     1 if normalize_patches else 0, float(var_constant), C.byref(h)))
        self._h = _ConvHandle(ctx, h.value)

    def apply(self, data):
        ds = _as_dataset(self.ctx, data)
        if not isinstance(ds, DeviceMatrix):
            ds = ds.materialize()
        return _ConvolvedImages(ds, self)


class SymmetricRectifier(Transformer):
    """Channels [0, C) = max(maxVal, v - alpha), [C, 2C) = max(maxVal, -v - alpha) (K/nodes/images/SymmetricRectifier.scala:7-32);
    on convolved images it becomes part of the convolution's epilogue."""

    def __init__(self, max_val: float = 0.0, alpha: float = 0.0):
        self.max_val, self.alpha = float(max_val), float(alpha)

    def apply(self, data):
        if isinstance(data, _ConvolvedImages) and data.rect is None and data.pool is None:
            return _ConvolvedImages(data.images, data.conv, (self.max_val, self.alpha), None)
        raise KeystoneError(-1, "SymmetricRectifier is implemented as the epilogue of a Convolver: apply it to a Convolver's output")


class Pooler(Transformer):
    """``new Pooler(stride, poolSize, identity, _.sum)`` (K/nodes/images/Pooler.scala:21-69; sum pooling of the pipeline,
    RandomPatchCifar.scala:61): fused into the convolution's epilogue."""

    def __init__(self, stride: int, pool_size: int):
        self.stride, self.pool_size = int(stride), int(pool_size)

    def apply(self, data):
        if isinstance(data, _ConvolvedImages) and data.rect is not None and data.pool is None:
            return _ConvolvedImages(data.images, data.conv, data.rect, (self.stride, self.pool_size))
        raise KeystoneError(-1, "Pooler is implemented as the epilogue of Convolver -> SymmetricRectifier: apply it to that chain's output")


class ImageVectorizer(Transformer):
    """``Image.toArray`` (K/nodes/images/ImageVectorizer.scala:12-16): forces the fused chain; rows are the vectorised images."""

    def apply(self, data):
        if isinstance(data, _ConvolvedImages):
            return data.materialize()
        return data


def images_to_matrix(images_xyc: np.ndarray) -> np.ndarray:
    """(n, x, y, c) image batch -> rows in ImageVectorizer order c + x*C + y*C*xDim (what Convolver expects)."""
    a = np.asarray(images_xyc)
    return np.ascontiguousarray(np.transpose(a, (0, 2, 1, 3)).reshape(a.shape[0], -1), dtype=np.float32)


def cifar_bytes_to_matrix(images_cxy: np.ndarray) -> np.ndarray:
    """CifarLoader's records (n, 3, 32, 32) -- RowColumnMajorByteArrayVectorizedImage: value (x, y, c) at y + x*yDim + c*yDim*xDim,
    K/utils/images/Image.scala:333-340 -- as Convolver input rows."""
    a = np.asarray(images_cxy)                       # [n][c][x][y]
    return images_to_matrix(np.transpose(a, (0, 2, 3, 1)))


class VectorCombiner(Transformer):
    """Concatenates the outputs of gathered branches (VectorCombiner.scala:11-14)."""

    def apply(self, parts: Sequence):
        if all(isinstance(p, LazyFeatures) for p in parts):
            out = parts[0]
            for p in parts[1:]:
                out = out.concat(p)
            return out
        ctx = next(p.ctx for p in parts if isinstance(p, Dataset))
        return ctx.matrix(np.concatenate([p.to_numpy(np.float32) if isinstance(p, Dataset) else np.asarray(p) for p in parts], axis=1))


class VectorSplitter:
    """Column blocks [j*blockSize, min(D, (j+1)*blockSize)) -- on the device a block is just a column offset, so
    this node only reports the boundaries (VectorSplitter.scala:15-25)."""

    def __init__(self, block_size: int, num_features_opt: Optional[int] = None):
        self.block_size, self.num_features_opt = block_size, num_features_opt

    def bounds(self, num_features: int):
        d = self.num_features_opt if self.num_features_opt is not None else num_features
        nb = int(math.ceil(d / float(self.block_size)))
        return [(j * self.block_size, min(d, (j + 1) * self.block_size)) for j in range(nb)]


class ClassLabelIndicatorsFromIntLabels(Transformer):
    def __init__(self, ctx: Context, num_classes: int):
        self.ctx, self.num_classes = ctx, num_classes

    def apply(self, labels):
        return self.ctx.labels_from_classes(np.asarray(labels), self.num_classes)


class MaxClassifier(Transformer):
    """argmax over scores.  Batches of predictions come back from the device as int32 class ids."""

    def apply(self, scores):
        if isinstance(scores, Dataset):
            scores = scores.to_numpy(np.float32)
        return np.argmax(np.asarray(scores), axis=-1).astype(np.int32)


# ------------------------------------------------------------------------------------------
class _ModelHandle:
    """Owns one model handle of the library (and with it the pinned host mirror the arrays below point into)."""

    def __init__(self, ctx: Context, handle: int):
        self.ctx, self.handle = ctx, handle

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                lib().ks_model_destroy(self.ctx.handle, self.handle)
        except Exception:
            pass


class _HostView:
    """Array-interface holder for a block of the model's pinned host mirror; numpy keeps it (and through it the model handle
    that owns the memory) alive as the array's base.  It references the handle object, not the mapper: no reference cycle,
    so dropping the mapper and its arrays frees the model at once."""

    def __init__(self, owner, ptr: int, shape, order: str):
        self.owner = owner
        strides = None
        if order == "F" and len(shape) == 2:
            strides = (8, 8 * shape[0])
        self.__array_interface__ = {"version": 3, "shape": tuple(shape), "typestr": "<f8", "data": (ptr, True), "strides": strides}


class BlockLinearMapper(Transformer):
    """Fitted model: xs (per-block (rows_j x k) matrices), blockSize, optional intercept and feature means."""

    def __init__(self, ctx: Context, handle: int):
        self.ctx, self.handle = ctx, handle
        self._owner = _ModelHandle(ctx, handle)
        nb, k, bs = C.c_int32(0), C.c_int64(0), C.c_int32(0)
        check(ctx.handle, lib().ks_model_num_blocks(ctx.handle, handle, C.byref(nb), C.byref(k), C.byref(bs)))
        self.num_blocks, self.k, self.block_size = nb.value, k.value, bs.value
        self._xs = None

    @classmethod
    def from_arrays(cls, ctx: Context, xs: Sequence[np.ndarray], block_size: int, b_opt: Optional[np.ndarray] = None,
                    feature_means: Optional[Sequence[np.ndarray]] = None) -> "BlockLinearMapper":
        """new BlockLinearMapper(xs, blockSize, bOpt, featureScalersOpt) (BlockLinearMapper.scala:22-27)."""
        xs_f = [np.asfortranarray(np.asarray(x, dtype=np.float64)) for x in xs]
        k = xs_f[0].shape[1]
        ptrs = (C.POINTER(C.c_double) * len(xs_f))(*[x.ctypes.data_as(C.POINTER(C.c_double)) for x in xs_f])
        rows = (C.c_int64 * len(xs_f))(*[x.shape[0] for x in xs_f])
        bb = None if b_opt is None else np.ascontiguousarray(b_opt, dtype=np.float64)
        mptr, means_c = None, None
        if feature_means is not None:
            means_c = [np.ascontiguousarray(m, dtype=np.float64) for m in feature_means]
            mptr = (C.POINTER(C.c_double) * len(means_c))(*[m.ctypes.data_as(C.POINTER(C.c_double)) for m in means_c])
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_model_from_host(ctx.handle, ptrs, rows, len(xs_f), k,
                                                    None if bb is None else bb.ctypes.data_as(C.c_void_p), mptr, block_size, C.byref(h)))
        return cls(ctx, h.value)

    # ---- model state (fp64, Breeze layouts) ----
    # The fit mirrors every finished block into pinned host memory while it is still running (ks_model_host_view); the
    # arrays below are read-only views of that mirror (no copy) and keep this mapper alive through their base object.
    def _view(self, ptr: int, shape, order: str) -> np.ndarray:
        return np.asarray(_HostView(self._owner, ptr, shape, order))

    def _block(self, j: int):
        rows = C.c_int64(0)
        check(self.ctx.handle, lib().ks_model_block_rows(self.ctx.handle, self.handle, j, C.byref(rows)))
        wp, mp = C.c_void_p(0), C.c_void_p(0)
        check(self.ctx.handle, lib().ks_model_host_view(self.ctx.handle, self.handle, j, C.byref(wp), C.byref(mp), None))
        W = self._view(wp.value, (rows.value, self.k), "F")
        mean = self._view(mp.value, (rows.value,), "C") if mp.value else None
        return W, mean

    @property
    def xs(self) -> List[np.ndarray]:
        if self._xs is None:
            self._xs = [self._block(j) for j in range(self.num_blocks)]
        return [w for w, _ in self._xs]

    @property
    def feature_means(self) -> Optional[List[np.ndarray]]:
        _ = self.xs
        return None if self._xs[0][1] is None else [m for _, m in self._xs]

    @property
    def b_opt(self) -> Optional[np.ndarray]:
        bp = C.c_void_p(0)
        check(self.ctx.handle, lib().ks_model_host_view(self.ctx.handle, self.handle, 0, None, None, C.byref(bp)))
        return self._view(bp.value, (self.k,), "C") if bp.value else None

    # ---- persistence (replaces the Java-serialised FittedPipeline, K/workflow/FittedPipeline.scala:18-22) ----
    def save(self, path: str) -> None:
        check(self.ctx.handle, lib().ks_model_save(self.ctx.handle, self.handle, path.encode()))

    @classmethod
    def load(cls, ctx: Context, path: str) -> "BlockLinearMapper":
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_model_load(ctx.handle, path.encode(), C.byref(h)))
        return cls(ctx, h.value)

    # ---- apply ----
    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 1
        ds = _as_dataset(self.ctx, data)
        f, x, rfs, n = feature_source_args(ds)
        h = C.c_int64(0)
        check(self.ctx.handle, lib().ks_model_apply(self.ctx.handle, self.handle, f, x, rfs, n, C.byref(h)))
        out = DeviceMatrix(self.ctx, h.value, ds.rows, self.k)
        return out.to_numpy()[0] if single else out

    def apply_argmax(self, data) -> np.ndarray:
        """apply followed by MaxClassifier, fused on the device."""
        ds = _as_dataset(self.ctx, data)
        f, x, rfs, n = feature_source_args(ds)
        out = np.empty(ds.rows, dtype=np.int32)
        check(self.ctx.handle, lib().ks_model_apply_argmax(self.ctx.handle, self.handle, f, x, rfs, n, out.ctypes.data_as(C.c_void_p)))
        return out

    def applyAndEvaluate(self, data, evaluator) -> None:
        """Calls ``evaluator(cumulative predictions incl. intercept)`` after every block (BlockLinearMapper.scala:95-137)."""
        ds = _as_dataset(self.ctx, data)
        f, x, rfs, n = feature_source_args(ds)
        for j in range(self.num_blocks):
            h = C.c_int64(0)
            check(self.ctx.handle, lib().ks_model_apply_partial(self.ctx.handle, self.handle, f, x, rfs, n, j, C.byref(h)))
            evaluator(DeviceMatrix(self.ctx, h.value, ds.rows, self.k))

    def compute_cost(self, data, labels, lam: float) -> float:
        """BlockLeastSquaresEstimator.computeCost (BlockLinearMapper.scala:142-187)."""
        ds = _as_dataset(self.ctx, data)
        lb = _as_dataset(self.ctx, labels)
        f, x, rfs, n = feature_source_args(ds)
        out = C.c_double(0)
        check(self.ctx.handle, lib().ks_model_cost(self.ctx.handle, self.handle, f, x, rfs, n, lb.handle, lam, C.byref(out)))
        return out.value

class LinearMapper(BlockLinearMapper):
    """LinearMapper(x, bOpt, featureScaler) (LinearMapper.scala:18-63): one weight matrix and one mean vector.  A model the
    library stores in feature blocks (DenseLBFGSwithL2 streams its features block by block) is the same mapper: ``x`` and
    ``feature_means`` join the blocks in feature order."""

    @classmethod
    def from_arrays(cls, ctx: Context, x: np.ndarray, b_opt=None, feature_mean=None):  # type: ignore[override]
        x = np.asarray(x, dtype=np.float64)
        return super().from_arrays(ctx, [x], x.shape[0], b_opt, None if feature_mean is None else [feature_mean])

    @property
    def x(self) -> np.ndarray:
        xs = self.xs
        return xs[0] if len(xs) == 1 else np.concatenate(xs, 0)

    @property
    def feature_means(self) -> Optional[List[np.ndarray]]:
        """[mean] (one vector over all features), or None: StandardScalerModel's mean, as the reference's featureScaler."""
        means = super().feature_means
        if means is None or len(means) == 1:
            return means
        return [np.concatenate(means)]


class BlockLeastSquaresEstimator(LabelEstimator, WeightedNode):
    def __init__(self, block_size: int, num_iter: int, lam: float = 0.0, num_features_opt: Optional[int] = None,
                 ctx: Optional[Context] = None, precision: str = "default"):
        """precision (KS_PRECISION_* of include/keystone_b200.h): "default" = the context's setting (initially the parity mode),
        "f16x2" / "parity" = split operands (hi + lo per MMA operand, >= 21 bits), "f16" = fp16 operands for the three big
        GEMMs on generated cosine features (10-bit mantissa, the fastest), "tf32" = one tf32 MMA per product."""
        self.block_size, self.num_iter, self.lam, self.num_features_opt, self.ctx = block_size, num_iter, lam, num_features_opt, ctx
        if precision not in _capi.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_capi.PRECISIONS)}")
        self.precision = precision
        self.weight = 3 * num_iter + 1  # BlockLinearMapper.scala:204

    def fit(self, data, labels) -> BlockLinearMapper:
        ds = _as_dataset(self.ctx, data)
        ctx = ds.ctx
        lb = _as_dataset(ctx, labels)
        f, x, rfs, n = feature_source_args(ds)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_blockls_fit(ctx.handle, f, x, rfs, n, lb.handle, self.block_size, self.num_iter, self.lam,
                                                self.num_features_opt or 0, _capi.PRECISIONS[self.precision], C.byref(h)))
        return BlockLinearMapper(ctx, h.value)

    def cost(self, n: int, d: int, k: int, sparsity: float, num_machines: int, cpu_weight: float, mem_weight: float,
             network_weight: float) -> float:
        """CostModel.cost (BlockLinearMapper.scala:268-282)."""
        flops = float(n) * d * (self.block_size + k) / num_machines
        bytes_scanned = float(n) * d / num_machines + float(d) * k
        network = 2.0 * (float(d) * (self.block_size + k)) * math.log(num_machines) / math.log(2.0)
        return self.num_iter * (max(cpu_weight * flops, mem_weight * bytes_scanned) + network_weight * network)


class BlockWeightedLeastSquaresEstimator(LabelEstimator, WeightedNode):
    def __init__(self, block_size: int, num_iter: int, lam: float, mixture_weight: float,
                 num_features_opt: Optional[int] = None, ctx: Optional[Context] = None, precision: str = "default"):
        self.block_size, self.num_iter, self.lam, self.mixture_weight = block_size, num_iter, lam, mixture_weight
        self.num_features_opt, self.ctx = num_features_opt, ctx
        if precision not in _capi.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_capi.PRECISIONS)}")
        self.precision = precision
        self.weight = 3 * num_iter + 1  # BlockWeightedLeastSquares.scala:44

    def fit(self, data, labels) -> BlockLinearMapper:
        ds = _as_dataset(self.ctx, data)
        ctx = ds.ctx
        lb = _as_dataset(ctx, labels)
        f, x, rfs, n = feature_source_args(ds)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_blockwls_fit(ctx.handle, f, x, rfs, n, lb.handle, self.block_size, self.num_iter, self.lam,
                                                 self.mixture_weight, self.num_features_opt or 0, _capi.PRECISIONS[self.precision],
                                                 C.byref(h)))
        return BlockLinearMapper(ctx, h.value)


class LinearMapEstimator(LabelEstimator):
    """Exact centred normal equations; computes in the context's precision (``ctx.set_option("precision", ...)``, initially the
    split-operand parity mode)."""

    def __init__(self, lam: Optional[float] = None, ctx: Optional[Context] = None):
        self.lam, self.ctx = lam, ctx

    def fit(self, data, labels) -> LinearMapper:
        ds = _as_dataset(self.ctx, data)
        if not isinstance(ds, DeviceMatrix):
            ds = ds.materialize()
        ctx = ds.ctx
        lb = _as_dataset(ctx, labels)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_linear_map_fit(ctx.handle, ds.handle, lb.handle, 0 if self.lam is None else 1,
                                                   0.0 if self.lam is None else float(self.lam), C.byref(h)))
        return LinearMapper(ctx, h.value)


class LeastSquaresDenseGradient:
    """The least-squares gradient of dense L-BFGS (K/nodes/learning/Gradient.scala:29-53): (A W - Y) and A^T (A W - Y).  A marker:
    the device computes it inside ``DenseLBFGSwithL2.fit``."""


class DenseLBFGSwithL2(LabelEstimator, WeightedNode):
    """``new DenseLBFGSwithL2(gradient, fitIntercept, numCorrections, convergenceTol, numIterations, regParam)``
    (K/nodes/learning/LBFGS.scala:135-192) on the device: minimises |A_c W - Y_c|^2 / (2N) + regParam / 2 |W|^2 from W = 0.

    Each step is the exact minimiser along the two-loop L-BFGS direction (the reference's Breeze line search is not
    reproduced, DESIGN.md section 14), so the iterates differ from the reference's while the minimiser is the same.  The fit
    stops after ``num_iterations`` steps or, with ``convergence_tol`` > 0, once max(last 10 losses) - f <= tol |f| or
    max |g| <= max(tol |f|, 1e-8).  After a fit, ``loss_history`` holds f(W_0) .. f(W_T), ``iterations`` T and
    ``stop_reason`` the rule that ended it.  ``precision`` as in ``BlockLeastSquaresEstimator``."""

    def __init__(self, gradient=None, fit_intercept: bool = True, num_corrections: int = 10, convergence_tol: float = 1e-4,
                 num_iterations: int = 100, reg_param: float = 0.0, ctx: Optional[Context] = None, precision: str = "default"):
        gradient = LeastSquaresDenseGradient() if gradient is None else gradient
        if not isinstance(gradient, LeastSquaresDenseGradient):
            raise ValueError("DenseLBFGSwithL2 supports LeastSquaresDenseGradient only")
        if int(num_corrections) < 1:
            raise ValueError("num_corrections must be >= 1")
        if int(num_iterations) < 1:
            raise ValueError("num_iterations must be >= 1")
        convergence_tol, reg_param = float(convergence_tol), float(reg_param)
        if not (convergence_tol >= 0.0 and math.isfinite(convergence_tol)):
            raise ValueError("convergence_tol must be finite and >= 0")
        if not (reg_param >= 0.0 and math.isfinite(reg_param)):
            raise ValueError("reg_param must be finite and >= 0")
        if precision not in _capi.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_capi.PRECISIONS)}")
        self.gradient, self.fit_intercept = gradient, bool(fit_intercept)
        self.num_corrections, self.convergence_tol, self.num_iterations = int(num_corrections), convergence_tol, int(num_iterations)
        self.reg_param, self.ctx, self.precision = reg_param, ctx, precision
        self.weight = self.num_iterations + 1  # LBFGS.scala:144
        self.loss_history: Optional[List[float]] = None
        self.iterations: Optional[int] = None
        self.stop_reason: Optional[str] = None
        self.stats: Optional[dict] = None

    def fit(self, data, labels) -> LinearMapper:
        """Collective with several ranks (data and labels: this rank's rows)."""
        ds = _as_dataset(self.ctx, data)
        ctx = ds.ctx
        lb = _as_dataset(ctx, labels)
        f, x, rfs, n = feature_source_args(ds)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_lbfgs_fit(ctx.handle, f, x, rfs, n, lb.handle, 1 if self.fit_intercept else 0, self.num_corrections,
                                              self.convergence_tol, self.num_iterations, self.reg_param, _capi.PRECISIONS[self.precision],
                                              C.byref(h)))
        model = LinearMapper(ctx, h.value)
        self.stats = ctx.last_fit_stats()
        self.loss_history = [float(v) for v in self.stats["loss_history"]]
        self.iterations, self.stop_reason = int(self.stats["iterations"]), self.stats["stop_reason"]
        return model

    def cost(self, n: int, d: int, k: int, sparsity: float, num_machines: int, cpu_weight: float, mem_weight: float,
             network_weight: float) -> float:
        """CostModel.cost (LBFGS.scala:175-191)."""
        flops = float(n) * d * k / num_machines
        bytes_scanned = float(n) * d / num_machines
        network = 2.0 * d * k * math.log(num_machines) / math.log(2.0)
        return self.num_iterations * (max(cpu_weight * flops, mem_weight * bytes_scanned) + network_weight * network)


class LeastSquaresEstimator(LabelEstimator, WeightedNode):
    """The reference's cost-model-driven solver choice (K/nodes/learning/LeastSquaresEstimator.scala:17-87): the four
    options' ``CostModel.cost`` formulas -- dense L-BFGS (K/nodes/learning/LBFGS.scala:175-191), sparse L-BFGS (:264-280),
    ``BlockLeastSquaresEstimator(1000, 3, lambda)`` (BlockLinearMapper.scala:268-282) and ``LinearMapEstimator(Some(lambda))``
    (LinearMapper.scala:100-115) -- with the reference's empirical weights; ``optimize`` returns the cheapest.

    ``fit`` runs the two direct solvers on the GPU.  When the cost model prefers an L-BFGS option, ``fit`` runs the GPU block
    solver instead and records both in ``selected`` / ``used``.  ``DenseLBFGSwithL2`` exists on the device too, but this routing
    is kept until measurements say where it beats the block solver (DESIGN.md section 14)."""

    def __init__(self, lam: float = 0.0, num_machines: Optional[int] = None, cpu_weight: float = 3.8e-4, mem_weight: float = 2.9e-1,
                 network_weight: float = 1.32, ctx: Optional[Context] = None):
        self.lam, self.num_machines, self.ctx = lam, num_machines, ctx
        self.cpu_weight, self.mem_weight, self.network_weight = cpu_weight, mem_weight, network_weight
        self.weight = 20 + 1          # default = DenseLBFGSwithL2(numIterations = 20): weight numIterations + 1 (LBFGS.scala)
        self.selected: Optional[str] = None
        self.used: Optional[str] = None

    @staticmethod
    def _sparse_lbfgs_cost(n, d, k, sparsity, m, cw, mw, nw, num_iterations: int = 20, sparse_overhead: float = 8.0):
        """SparseLBFGSwithL2.cost (LBFGS.scala:264-280)."""
        flops = float(n) * sparsity * d * k / m
        bytes_scanned = float(n) * d * sparsity / m
        network = 2.0 * d * k * math.log(m) / math.log(2.0)
        return num_iterations * (sparse_overhead * max(cw * flops, mw * bytes_scanned) + nw * network)

    def costs(self, n: int, d: int, k: int, sparsity: float, num_machines: int) -> dict:
        cw, mw, nw = self.cpu_weight, self.mem_weight, self.network_weight
        block = BlockLeastSquaresEstimator(1000, 3, self.lam)
        exact_flops = float(n) * d * (d + k) / num_machines
        exact_bytes = float(n) * d / num_machines + float(d) * d
        return {
            "dense_lbfgs": DenseLBFGSwithL2(num_iterations=20).cost(n, d, k, sparsity, num_machines, cw, mw, nw),
            "sparse_lbfgs": self._sparse_lbfgs_cost(n, d, k, sparsity, num_machines, cw, mw, nw),
            "block": block.cost(n, d, k, sparsity, num_machines, cw, mw, nw),
            "exact": max(cw * exact_flops, mw * exact_bytes) + nw * float(d) * (d + k),
        }

    def optimize(self, n: int, d: int, k: int, sparsity: float = 1.0, num_machines: Optional[int] = None) -> str:
        """``options.minBy(cost)`` (:83); ties resolve in the reference's option order."""
        m = num_machines or self.num_machines or 1
        c = self.costs(n, d, k, sparsity, m)
        self.selected = min(("dense_lbfgs", "sparse_lbfgs", "block", "exact"), key=lambda name: c[name])
        return self.selected

    def fit(self, data, labels) -> BlockLinearMapper:
        ds = _as_dataset(self.ctx, data)
        lb = _as_dataset(ds.ctx, labels)
        n_total = ds.rows * max(1, ds.ctx.world_size)
        choice = self.optimize(n_total, ds.cols, lb.cols, 1.0, self.num_machines or ds.ctx.world_size)
        if choice == "exact":
            self.used = "exact"
            return LinearMapEstimator(self.lam, ds.ctx).fit(ds, lb)
        self.used = "block"
        return BlockLeastSquaresEstimator(1000, 3, self.lam, ctx=ds.ctx).fit(ds, lb)


# ------------------------------------------------------------------------------------------ Gaussian-kernel ridge regression
class _KernelHandle:
    def __init__(self, ctx: Context, handle: int):
        self.ctx, self.handle = ctx, handle

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                lib().ks_gaussian_kernel_destroy(self.ctx.handle, self.handle)
        except Exception:
            pass


def _device_rows(ctx: Optional[Context], data) -> DeviceMatrix:
    ds = _as_dataset(ctx, data)
    return ds if isinstance(ds, DeviceMatrix) else ds.materialize()


class GaussianKernelGenerator(Estimator):
    """``new GaussianKernelGenerator(gamma, cacheKernel)`` (K/nodes/learning/KernelGenerator.scala:36-44):
    K(x, y) = exp(-gamma |x - y|^2).  ``cache_kernel`` is accepted for API parity and has no effect: kernel blocks are
    regenerated on the device whenever they are needed."""

    def __init__(self, gamma: float, cache_kernel: bool = False, ctx: Optional[Context] = None):
        gamma = float(gamma)
        if not (gamma > 0.0 and math.isfinite(gamma)):
            raise ValueError("gamma must be finite and > 0")
        self.gamma, self.cache_kernel, self.ctx = gamma, cache_kernel, ctx

    def fit(self, train) -> "GaussianKernelTransformer":
        """Collective with several ranks: every rank passes its training rows; the transformer holds all of them."""
        x = _device_rows(self.ctx, train)
        h = C.c_int64(0)
        check(x.ctx.handle, lib().ks_gaussian_kernel_create(x.ctx.handle, x.handle, self.gamma, C.byref(h)))
        return GaussianKernelTransformer(x.ctx, h.value, self.gamma)


class GaussianKernelTransformer(Transformer):
    """The fitted kernel (KernelGenerator.scala:84-119): the training rows of every rank, in rank order."""

    def __init__(self, ctx: Context, handle: int, gamma: float):
        self.ctx, self.handle, self.gamma = ctx, handle, gamma
        self._owner = _KernelHandle(ctx, handle)
        n, d = C.c_int64(0), C.c_int64(0)
        check(ctx.handle, lib().ks_gaussian_kernel_shape(ctx.handle, handle, C.byref(n), C.byref(d)))
        self.n_train, self.dim = n.value, d.value   # training rows over all ranks, their width

    def block(self, data, col0: int, cols: int) -> DeviceMatrix:
        """K(data, training rows [col0, col0 + cols)) as a device matrix."""
        x = _device_rows(self.ctx, data)
        h = C.c_int64(0)
        check(self.ctx.handle, lib().ks_gaussian_kernel_block(self.ctx.handle, self.handle, x.handle, int(col0), int(cols), C.byref(h)))
        return DeviceMatrix(self.ctx, h.value, x.rows, int(cols))

    def apply(self, data):
        """A dataset gives its KernelMatrix (lazy); a 1-D vector gives its kernel row against every training row."""
        if isinstance(data, np.ndarray) and data.ndim == 1:
            return self.block(np.asarray(data, dtype=np.float64)[None, :], 0, self.n_train).to_numpy()[0]
        return KernelMatrix(self, _device_rows(self.ctx, data))


class KernelMatrix:
    """BlockKernelMatrix (K/nodes/learning/KernelMatrix.scala:50-95): column blocks of K(data, training rows), generated on the
    device when asked for.  Column blocks are contiguous ranges of training rows."""

    def __init__(self, transformer: GaussianKernelTransformer, data: DeviceMatrix):
        self.transformer, self.data = transformer, data

    @staticmethod
    def _range(idxs: Sequence[int]):
        idx = np.asarray(list(idxs), dtype=np.int64)
        if idx.size == 0 or np.any(np.diff(idx) != 1):
            raise ValueError("column indices must be a non-empty contiguous ascending range")
        return int(idx[0]), int(idx.size)

    def __call__(self, col_idxs: Sequence[int]) -> DeviceMatrix:
        c0, n = self._range(col_idxs)
        return self.transformer.block(self.data, c0, n)

    def diag_block(self, idxs: Sequence[int]) -> np.ndarray:
        """K(data rows idxs, training rows idxs): the rows idxs of the column block idxs (this rank's data rows)."""
        c0, n = self._range(idxs)
        return self(idxs).to_numpy()[c0:c0 + n]

    def unpersist(self, col_idxs: Sequence[int]) -> None:
        """Nothing is cached."""


class KernelBlockLinearMapper(BlockLinearMapper):
    """``KernelBlockLinearMapper(model, blockSize, kernelTransformer, nTrain)`` (K/nodes/learning/KernelBlockLinearMapper.scala:
    28-89): predictions sum_j K(x, X_j) W_j on raw input rows.  Kernel models are not persisted (save / compute_cost /
    applyAndEvaluate raise)."""

    def __init__(self, ctx: Context, handle: int, kernel_transformer: GaussianKernelTransformer):
        super().__init__(ctx, handle)
        self.kernel_transformer = kernel_transformer

    @classmethod
    def from_arrays(cls, ctx: Context, xs: Sequence[np.ndarray], block_size: int,  # type: ignore[override]
                    kernel_transformer: GaussianKernelTransformer) -> "KernelBlockLinearMapper":
        xs_f = [np.asfortranarray(np.asarray(x, dtype=np.float64)) for x in xs]
        k = xs_f[0].shape[1]
        ptrs = (C.POINTER(C.c_double) * len(xs_f))(*[x.ctypes.data_as(C.POINTER(C.c_double)) for x in xs_f])
        rows = (C.c_int64 * len(xs_f))(*[x.shape[0] for x in xs_f])
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_kernel_model_from_host(ctx.handle, kernel_transformer.handle, ptrs, rows, len(xs_f), k, block_size,
                                                           C.byref(h)))
        return cls(ctx, h.value, kernel_transformer)

    @property
    def model(self) -> List[np.ndarray]:
        return self.xs


class KernelRidgeRegression(LabelEstimator):
    """``new KernelRidgeRegression(kernelGenerator, lambda, blockSize, numEpochs, blockPermuter, blocksBeforeCheckpoint)``
    (K/nodes/learning/KernelRidgeRegression.scala:37-84): block Gauss-Seidel on (K + lambda I) W = Y over contiguous blocks
    of training rows, no centring, no intercept.

    ``block_permuter``: a seed; each epoch visits the blocks in ``numpy.random.Generator(PCG64(seed)).permutation`` order (one
    draw per epoch).  Scala's ``Random.shuffle`` stream is not reproduced.  ``blocks_before_checkpoint`` is accepted for API
    parity and has no effect (there is no Spark lineage to truncate)."""

    def __init__(self, kernel_generator: GaussianKernelGenerator, lam: float, block_size: int, num_epochs: int,
                 block_permuter: Optional[int] = None, blocks_before_checkpoint: int = 25, ctx: Optional[Context] = None):
        if int(block_size) < 1:
            raise ValueError("block_size must be >= 1")
        if int(num_epochs) < 1:
            raise ValueError("num_epochs must be >= 1")
        lam = float(lam)
        if not (lam >= 0.0 and math.isfinite(lam)):
            raise ValueError("lam must be finite and >= 0")
        self.kernel_generator, self.lam, self.block_size, self.num_epochs = kernel_generator, lam, int(block_size), int(num_epochs)
        self.block_permuter, self.blocks_before_checkpoint, self.ctx = block_permuter, blocks_before_checkpoint, ctx

    def block_order(self, n_train: int) -> Optional[np.ndarray]:
        if self.block_permuter is None:
            return None
        nb = -(-n_train // self.block_size)
        rng = np.random.Generator(np.random.PCG64(self.block_permuter))
        return np.stack([rng.permutation(nb) for _ in range(self.num_epochs)]).astype(np.int32)

    def fit(self, data, labels) -> KernelBlockLinearMapper:
        """Collective with several ranks (data and labels: this rank's rows)."""
        x = _device_rows(self.ctx or self.kernel_generator.ctx, data)
        ctx = x.ctx
        lb = _device_rows(ctx, labels)
        transformer = self.kernel_generator.fit(x)
        order = self.block_order(transformer.n_train)
        optr = None if order is None else np.ascontiguousarray(order).ctypes.data_as(C.c_void_p)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_krr_fit(ctx.handle, transformer.handle, lb.handle, self.lam, self.block_size, self.num_epochs, optr,
                                            C.byref(h)))
        return KernelBlockLinearMapper(ctx, h.value, transformer)


class StandardScalerModel(Transformer):
    """(x - mean) [/ std] as a LinearMapper-free node is out of the hot path; the fits above centre internally
    (BlockLinearMapper.scala:224-232).  Kept for API parity: holds the statistics a fitted model reports."""

    def __init__(self, mean: np.ndarray, std: Optional[np.ndarray] = None):
        self.mean, self.std = mean, std
