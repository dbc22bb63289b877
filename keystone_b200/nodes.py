"""Node library of the hot path: same class names, constructor arguments and semantics as the
reference nodes; the bodies marshal to the C ABI (which launches the sm_90a kernels).

Reference classes (K/ = src/main/scala/keystoneml/):
  CosineRandomFeatures                K/nodes/stats/CosineRandomFeatures.scala:19-60
  StandardScaler / StandardScalerModel K/nodes/stats/StandardScaler.scala:16-59
  Windower, Cropper, RandomPatcher,   K/nodes/images/*.scala (image views, DESIGN.md section 21)
  CenterCornerPatcher, RandomImageTransformer
  Sampler                             K/nodes/stats/Sampling.scala
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
  SparseLBFGSwithL2                   K/nodes/learning/LBFGS.scala:208-281
  LeastSquaresSparseGradient          K/nodes/learning/Gradient.scala
  SparseLinearMapper                  K/nodes/learning/SparseLinearMapper.scala
  Densify                             K/nodes/util/Densify.scala
  LogisticRegressionEstimator / Model K/nodes/learning/LogisticRegressionModel.scala
  NaiveBayesEstimator / Model         K/nodes/learning/NaiveBayesModel.scala
  Trim, LowerCase, Tokenizer          K/nodes/nlp/StringUtils.scala (text front end, DESIGN.md section 23)
  NGramsFeaturizer                    K/nodes/nlp/ngrams.scala
  TermFrequency                       K/nodes/stats/TermFrequency.scala
  CommonSparseFeatures, AllSparseFeatures, SparseFeatureVectorizer   K/nodes/util/*.scala
  HashingTF, NGramsHashingTF          K/nodes/nlp/{HashingTF,NGramsHashingTF}.scala

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
from .context import (Context, Dataset, DeviceMatrix, LazyFeatures, NGramBatch, SparseMatrix, TermFrequencyBatch, TextBatch, TokenBatch,
                      _flatten_terms, _host_terms, feature_source_args)
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
    chunk when it is materialised (``ImageVectorizer`` / ``to_numpy``).  ``images`` is a device matrix of images or ``ImageViews``,
    whose views the launch gathers chunk by chunk."""

    def __init__(self, images, conv: "Convolver", rect=None, pool=None):
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
        if isinstance(self.images, ImageViews):
            v = self.images
            check(self.ctx.handle, lib().ks_convolver_apply_views(self.ctx.handle, self.conv._h.handle, v.source.matrix.handle, v.source.x_dim,
                                                                   v.source.y_dim, v.views.ctypes.data_as(C.c_void_p), v.rows, stride, size,
                                                                   float(max_val), float(alpha), C.byref(h)))
        else:
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
        if isinstance(data, ImageViews):
            if (data.x_dim, data.y_dim, data.channels) != (self.x_dim, self.y_dim, self.ch):
                raise KeystoneError(-1, "Convolver: the views' size does not match the Convolver's image size")
            return _ConvolvedImages(data, self)
        ds = _as_dataset(self.ctx, data.matrix if isinstance(data, ImageBatch) else data)
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
        if isinstance(data, (_ConvolvedImages, ImageViews)):
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


def _as_sparse(ctx: Optional[Context], data) -> SparseMatrix:
    if isinstance(data, SparseMatrix):
        return data
    if isinstance(data, Dataset):
        raise KeystoneError(-1, f"a sparse node needs a SparseMatrix, not {type(data).__name__}")
    if ctx is None:
        raise KeystoneError(-1, "host sparse input needs a Context (pass ctx= to the node)")
    return ctx.sparse(data)


class LeastSquaresSparseGradient:
    """The least-squares gradient of sparse L-BFGS (K/nodes/learning/Gradient.scala): (A W - Y) and A^T (A W - Y) over sparse rows.
    A marker: the device computes it inside ``SparseLBFGSwithL2.fit``."""


class SparseLinearMapper(LinearMapper):
    """SparseLinearMapper(x, bOpt) (K/nodes/learning/SparseLinearMapper.scala): x (d x k) and an optional intercept, applied to
    sparse rows as A x + b; it carries no feature means.  ``SparseLinearMapper(x, b_opt, ctx)`` builds it from host arrays (stored
    in feature blocks of min(d, 4096) rows, as the fit stores it); ``SparseLinearMapper(ctx, handle)`` wraps a fitted or loaded
    model handle."""

    def __init__(self, x, b_opt=None, ctx: Optional[Context] = None):
        if isinstance(x, Context):   # (ctx, handle)
            super().__init__(x, int(b_opt))
            return
        if ctx is None:
            raise KeystoneError(-1, "SparseLinearMapper from host arrays needs a Context (pass ctx=)")
        x = np.asfortranarray(np.asarray(x, dtype=np.float64))
        if x.ndim != 2 or x.shape[0] < 1 or x.shape[1] < 1:
            raise ValueError("x must be a non-empty d x k matrix")
        bs = min(x.shape[0], 4096)
        blocks = [np.asfortranarray(x[i:i + bs]) for i in range(0, x.shape[0], bs)]
        ptrs = (C.POINTER(C.c_double) * len(blocks))(*[w.ctypes.data_as(C.POINTER(C.c_double)) for w in blocks])
        rows = (C.c_int64 * len(blocks))(*[w.shape[0] for w in blocks])
        bb = None if b_opt is None else np.ascontiguousarray(b_opt, dtype=np.float64)
        if bb is not None and bb.shape != (x.shape[1],):
            raise ValueError("b_opt must hold k values")
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_model_from_host(ctx.handle, ptrs, rows, len(blocks), x.shape[1],
                                                    None if bb is None else bb.ctypes.data_as(C.c_void_p), None, bs, C.byref(h)))
        super().__init__(ctx, h.value)

    def apply(self, data):
        """A W + b for the rows of a ``SparseMatrix`` (or a host sparse object), fp64 on the device, rounded once to fp32."""
        sm = _as_sparse(self.ctx, data)
        h = C.c_int64(0)
        check(self.ctx.handle, lib().ks_model_apply_sparse(self.ctx.handle, self.handle, sm.handle, C.byref(h)))
        return DeviceMatrix(self.ctx, h.value, sm.rows, self.k)


class Densify(Transformer):
    """Densify (K/nodes/util/Densify.scala): a ``SparseMatrix`` as a new fp32 ``DeviceMatrix``; repeated entries are summed in fp64
    and rounded once."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    def apply(self, data) -> DeviceMatrix:
        sm = _as_sparse(self.ctx, data)
        h = C.c_int64(0)
        check(sm.ctx.handle, lib().ks_sparse_densify(sm.ctx.handle, sm.handle, C.byref(h)))
        return DeviceMatrix(sm.ctx, h.value, sm.rows, sm.cols)


class SparseLBFGSwithL2(LabelEstimator, WeightedNode):
    """``new SparseLBFGSwithL2(gradient, fitIntercept, numCorrections, convergenceTol, numIterations, regParam, sparseOverhead)``
    (K/nodes/learning/LBFGS.scala:208-281) on the device, in fp64 throughout.

    The data is not centred.  With ``fit_intercept`` the rows get an implicit column of ones (never stored) and the fit minimises
    f = |[A 1][W; b] - Y|^2 / (2N) + regParam / 2 |[W; b]|^2 from zero, returning ``SparseLinearMapper(W, b)``; without it, W alone.
    The bias is regularised in both f and its gradient: the reference's gradient regularises it (LBFGS.scala:117) while its loss
    leaves it out (:106-113), so this fit converges to the zero of the reference's gradient with the f whose gradient that is.  At
    regParam = 0 (the default) the two agree.  The direction, exact step and stop rules are those of ``DenseLBFGSwithL2``
    (DESIGN.md sections 14 and 20); ``loss_history``, ``iterations``, ``stop_reason`` and ``stats`` are set after a fit.  One rank
    fitting the same input twice gets a bit-identical model."""

    def __init__(self, gradient=None, fit_intercept: bool = True, num_corrections: int = 10, convergence_tol: float = 1e-4,
                 num_iterations: int = 100, reg_param: float = 0.0, sparse_overhead: float = 8.0, ctx: Optional[Context] = None):
        gradient = LeastSquaresSparseGradient() if gradient is None else gradient
        if not isinstance(gradient, LeastSquaresSparseGradient):
            raise ValueError("SparseLBFGSwithL2 supports LeastSquaresSparseGradient only")
        if int(num_corrections) < 1:
            raise ValueError("num_corrections must be >= 1")
        if int(num_iterations) < 1:
            raise ValueError("num_iterations must be >= 1")
        convergence_tol, reg_param = float(convergence_tol), float(reg_param)
        if not (convergence_tol >= 0.0 and math.isfinite(convergence_tol)):
            raise ValueError("convergence_tol must be finite and >= 0")
        if not (reg_param >= 0.0 and math.isfinite(reg_param)):
            raise ValueError("reg_param must be finite and >= 0")
        self.gradient, self.fit_intercept = gradient, bool(fit_intercept)
        self.num_corrections, self.convergence_tol, self.num_iterations = int(num_corrections), convergence_tol, int(num_iterations)
        self.reg_param, self.sparse_overhead, self.ctx = reg_param, float(sparse_overhead), ctx
        self.weight = self.num_iterations + 1  # LBFGS.scala:220
        self.loss_history: Optional[List[float]] = None
        self.iterations: Optional[int] = None
        self.stop_reason: Optional[str] = None
        self.stats: Optional[dict] = None

    def fit(self, data, labels) -> SparseLinearMapper:
        """Collective with several ranks (data and labels: this rank's rows)."""
        sm = _as_sparse(self.ctx, data)
        ctx = sm.ctx
        lb = _as_dataset(ctx, labels)
        if not isinstance(lb, DeviceMatrix):
            raise KeystoneError(-1, "labels must be a DeviceMatrix or a 2-D array")
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_sparse_lbfgs_fit(ctx.handle, sm.handle, lb.handle, 1 if self.fit_intercept else 0, self.num_corrections,
                                                     self.convergence_tol, self.num_iterations, self.reg_param, C.byref(h)))
        model = SparseLinearMapper(ctx, h.value)
        self.stats = ctx.last_fit_stats()
        self.loss_history = [float(v) for v in self.stats["loss_history"]]
        self.iterations, self.stop_reason = int(self.stats["iterations"]), self.stats["stop_reason"]
        return model

    def cost(self, n: int, d: int, k: int, sparsity: float, num_machines: int, cpu_weight: float, mem_weight: float,
             network_weight: float) -> float:
        """CostModel.cost (LBFGS.scala:264-280)."""
        flops = float(n) * sparsity * d * k / num_machines
        bytes_scanned = float(n) * d * sparsity / num_machines
        network = 2.0 * d * k * math.log(num_machines) / math.log(2.0)
        return self.num_iterations * (self.sparse_overhead * max(cpu_weight * flops, mem_weight * bytes_scanned)
                                      + network_weight * network)


# ------------------------------------------------------------------------------------------ classifiers (DESIGN.md section 22)
def _classifier_input(ctx: Optional[Context], data):
    """A fit's feature source: (features handle or 0, sparse handle or 0, context, rows, columns).  Lazy sources are refused."""
    if isinstance(data, SparseMatrix):
        return 0, data.handle, data.ctx, data.rows, data.cols
    if isinstance(data, Dataset) and not isinstance(data, DeviceMatrix):
        raise KeystoneError(-1, f"{type(data).__name__} is not accepted here: pass a DeviceMatrix or a SparseMatrix")
    if not isinstance(data, Dataset) and hasattr(data, "indptr"):
        data = _as_sparse(ctx, data)
        return 0, data.handle, data.ctx, data.rows, data.cols
    dm = _as_dataset(ctx, data)
    return dm.handle, 0, dm.ctx, dm.rows, dm.cols


def _class_labels(labels, rows: int) -> np.ndarray:
    y = np.asarray(labels)
    if y.ndim != 1 or y.shape[0] != rows:
        raise KeystoneError(-1, f"labels must be a 1-D array of {rows} class ids")
    if y.size and not np.all(y == np.round(y)):
        raise KeystoneError(-1, "labels must be integer class ids")
    return np.ascontiguousarray(y, dtype=np.int32)


def _first_max(scores: np.ndarray) -> np.ndarray:
    return np.argmax(scores, axis=-1).astype(np.float64)


class LogisticRegressionModel(BlockLinearMapper):
    """LogisticRegressionModel (K/nodes/learning/LogisticRegressionModel.scala): MLlib's model without an intercept, stored as an
    ordinary d x k model whose column 0 is zero (the pivot class).  ``apply`` returns float64 class ids, MLlib's ``predict``: the
    first maximum of [0, x . w_1, ..., x . w_(k-1)].  ``weights`` is MLlib's flattened (k-1) * d vector, class-major."""

    intercept = 0.0

    def __init__(self, ctx: Context, handle: int):
        super().__init__(ctx, handle)

    @property
    def num_classes(self) -> int:
        return self.k

    @property
    def num_features(self) -> int:
        return int(sum(w.shape[0] for w in self.xs))

    @property
    def weights(self) -> np.ndarray:
        W = np.concatenate(self.xs, 0)
        return np.ascontiguousarray(W[:, 1:].T).ravel()

    def apply(self, data):
        if isinstance(data, np.ndarray) and data.ndim == 1:
            return float(self.apply(data[None, :])[0])
        if isinstance(data, SparseMatrix) or (not isinstance(data, Dataset) and hasattr(data, "indptr")):
            sm = _as_sparse(self.ctx, data)
            h = C.c_int64(0)
            check(self.ctx.handle, lib().ks_model_apply_sparse(self.ctx.handle, self.handle, sm.handle, C.byref(h)))
            return _first_max(DeviceMatrix(self.ctx, h.value, sm.rows, self.k).to_numpy(np.float32))
        return self.apply_argmax(data).astype(np.float64)


class LogisticRegressionEstimator(LabelEstimator):
    """``LogisticRegressionEstimator(numClasses, regParam, numIters, convergenceTol, numFeatures)``
    (K/nodes/learning/LogisticRegressionModel.scala) on the device, fp64 throughout: MLlib's LogisticGradient with SquaredL2Updater,
    no intercept, no feature scaling, by L-BFGS (10 corrections) with a strong-Wolfe line search modelled on Breeze's
    (DESIGN.md section 22).  ``convergence_tol`` is honoured (the reference does not pass it on).  ``fit(data, labels)`` takes a
    ``DeviceMatrix`` or ``SparseMatrix`` (this rank's rows) and the rank's class ids; collective with several ranks.
    ``loss_history``, ``iterations``, ``stop_reason``, ``line_search_evals`` and ``stats`` are set after a fit."""

    def __init__(self, num_classes: int, reg_param: float = 0.0, num_iters: int = 100, convergence_tol: float = 1e-4,
                 num_features: int = -1, ctx: Optional[Context] = None):
        if int(num_classes) < 2:
            raise ValueError("num_classes must be >= 2")
        if int(num_iters) < 1:
            raise ValueError("num_iters must be >= 1")
        reg_param, convergence_tol = float(reg_param), float(convergence_tol)
        if not (reg_param >= 0.0 and math.isfinite(reg_param)):
            raise ValueError("reg_param must be finite and >= 0")
        if not (convergence_tol >= 0.0 and math.isfinite(convergence_tol)):
            raise ValueError("convergence_tol must be finite and >= 0")
        self.num_classes, self.reg_param, self.num_iters = int(num_classes), reg_param, int(num_iters)
        self.convergence_tol, self.num_features, self.ctx = convergence_tol, int(num_features), ctx
        self.loss_history: Optional[List[float]] = None
        self.iterations: Optional[int] = None
        self.stop_reason: Optional[str] = None
        self.line_search_evals: Optional[List[int]] = None
        self.stats: Optional[dict] = None

    def fit(self, data, labels) -> LogisticRegressionModel:
        f, s, ctx, rows, cols = _classifier_input(self.ctx, data)
        if self.num_features not in (-1, cols):
            raise KeystoneError(-1, f"num_features is {self.num_features} but the data has {cols} columns")
        y = _class_labels(labels, rows)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_logistic_fit(ctx.handle, f, s, y.ctypes.data_as(C.c_void_p), rows, self.num_classes, self.reg_param,
                                                 self.num_iters, self.convergence_tol, C.byref(h)))
        model = LogisticRegressionModel(ctx, h.value)
        self.stats = ctx.last_fit_stats()
        self.loss_history = [float(v) for v in self.stats["loss_history"]]
        self.iterations, self.stop_reason = int(self.stats["iterations"]), self.stats["stop_reason"]
        self.line_search_evals = [int(v) for v in self.stats["line_search_evals"]]
        return model


class NaiveBayesModel(BlockLinearMapper):
    """NaiveBayesModel(labels, pi, theta) (K/nodes/learning/NaiveBayesModel.scala): ``apply`` gives the log-posteriors
    x theta^T + pi (follow it with ``MaxClassifier``).  Stored as an ordinary model, W = theta^T (d x k) in feature blocks of
    min(d, 4096) rows and intercept pi.  ``NaiveBayesModel(labels, pi, theta, ctx=ctx)`` builds it from host arrays;
    ``NaiveBayesModel(ctx, handle)`` wraps a fitted or loaded model (labels 0 .. k-1)."""

    def __init__(self, labels, pi=None, theta=None, ctx: Optional[Context] = None):
        if isinstance(labels, Context):   # (ctx, handle)
            super().__init__(labels, int(pi))
            self.labels = np.arange(self.k)
            return
        if ctx is None:
            raise KeystoneError(-1, "NaiveBayesModel from host arrays needs a Context (pass ctx=)")
        pi = np.ascontiguousarray(pi, dtype=np.float64)
        theta = np.asarray(theta, dtype=np.float64)
        if theta.ndim != 2 or pi.shape != (theta.shape[0],) or theta.shape[1] < 1 or len(labels) != theta.shape[0]:
            raise ValueError("theta must be k x d, with k values in pi and in labels")
        W = np.asfortranarray(theta.T)
        bs = min(W.shape[0], 4096)
        blocks = [np.asfortranarray(W[i:i + bs]) for i in range(0, W.shape[0], bs)]
        ptrs = (C.POINTER(C.c_double) * len(blocks))(*[w.ctypes.data_as(C.POINTER(C.c_double)) for w in blocks])
        rows = (C.c_int64 * len(blocks))(*[w.shape[0] for w in blocks])
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_model_from_host(ctx.handle, ptrs, rows, len(blocks), W.shape[1], pi.ctypes.data_as(C.c_void_p), None,
                                                    bs, C.byref(h)))
        super().__init__(ctx, h.value)
        self.labels = np.asarray(labels)

    @property
    def pi(self) -> np.ndarray:
        return np.array(self.b_opt)

    @property
    def theta(self) -> np.ndarray:
        return np.ascontiguousarray(np.concatenate(self.xs, 0).T)

    def apply(self, data):
        if isinstance(data, SparseMatrix) or (not isinstance(data, Dataset) and hasattr(data, "indptr")):
            sm = _as_sparse(self.ctx, data)
            h = C.c_int64(0)
            check(self.ctx.handle, lib().ks_model_apply_sparse(self.ctx.handle, self.handle, sm.handle, C.byref(h)))
            return DeviceMatrix(self.ctx, h.value, sm.rows, self.k)
        return super().apply(data)


class NaiveBayesEstimator(LabelEstimator):
    """``NaiveBayesEstimator(numClasses, lambda)`` (K/nodes/learning/NaiveBayesModel.scala), MLlib's multinomial NaiveBayes.train on
    the device: pi_c = log(n_c + lam) - log(N + k lam), theta_cj = log(S_cj + lam) - log(sum_j S_cj + d lam) with S_cj the sum of
    feature j over class c.  Negative or NaN feature values, labels outside [0, num_classes) and classes with no rows are rejected
    (on every rank).  ``fit(data, labels)`` as for ``LogisticRegressionEstimator``; collective with several ranks."""

    def __init__(self, num_classes: int, lam: float = 1.0, ctx: Optional[Context] = None):
        if int(num_classes) < 2:
            raise ValueError("num_classes must be >= 2")
        lam = float(lam)
        if not (lam >= 0.0 and math.isfinite(lam)):
            raise ValueError("lam must be finite and >= 0")
        self.num_classes, self.lam, self.ctx = int(num_classes), lam, ctx
        self.stats: Optional[dict] = None

    def fit(self, data, labels) -> NaiveBayesModel:
        f, s, ctx, rows, _ = _classifier_input(self.ctx, data)
        y = _class_labels(labels, rows)
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_naive_bayes_fit(ctx.handle, f, s, y.ctypes.data_as(C.c_void_p), rows, self.num_classes, self.lam,
                                                    C.byref(h)))
        self.stats = ctx.last_fit_stats()
        return NaiveBayesModel(ctx, h.value)


class LeastSquaresEstimator(LabelEstimator, WeightedNode):
    """The reference's cost-model-driven solver choice (K/nodes/learning/LeastSquaresEstimator.scala:17-87): the four
    options' ``CostModel.cost`` formulas -- dense L-BFGS (K/nodes/learning/LBFGS.scala:175-191), sparse L-BFGS (:264-280),
    ``BlockLeastSquaresEstimator(1000, 3, lambda)`` (BlockLinearMapper.scala:268-282) and ``LinearMapEstimator(Some(lambda))``
    (LinearMapper.scala:100-115) -- with the reference's empirical weights; ``optimize`` returns the cheapest.

    ``fit`` runs the two direct solvers on the GPU.  When the cost model prefers dense L-BFGS, ``fit`` runs the GPU block
    solver instead and records both in ``selected`` / ``used``.  ``DenseLBFGSwithL2`` exists on the device too, but this routing
    is kept until measurements say where it beats the block solver (DESIGN.md section 14).

    A ``SparseMatrix`` input is costed with sparsity = local nnz / (local rows x d).  ``sparse_lbfgs`` runs
    ``SparseLBFGSwithL2(num_iterations=20, reg_param=lam)`` on it; every other choice densifies it first
    (LeastSquaresEstimator.scala:44-50): ``exact`` then runs ``LinearMapEstimator``, ``block`` and ``dense_lbfgs`` the block
    solver."""

    def __init__(self, lam: float = 0.0, num_machines: Optional[int] = None, cpu_weight: float = 3.8e-4, mem_weight: float = 2.9e-1,
                 network_weight: float = 1.32, ctx: Optional[Context] = None):
        self.lam, self.num_machines, self.ctx = lam, num_machines, ctx
        self.cpu_weight, self.mem_weight, self.network_weight = cpu_weight, mem_weight, network_weight
        self.weight = 20 + 1          # default = DenseLBFGSwithL2(numIterations = 20): weight numIterations + 1 (LBFGS.scala)
        self.selected: Optional[str] = None
        self.used: Optional[str] = None

    def costs(self, n: int, d: int, k: int, sparsity: float, num_machines: int) -> dict:
        cw, mw, nw = self.cpu_weight, self.mem_weight, self.network_weight
        block = BlockLeastSquaresEstimator(1000, 3, self.lam)
        exact_flops = float(n) * d * (d + k) / num_machines
        exact_bytes = float(n) * d / num_machines + float(d) * d
        return {
            "dense_lbfgs": DenseLBFGSwithL2(num_iterations=20).cost(n, d, k, sparsity, num_machines, cw, mw, nw),
            "sparse_lbfgs": SparseLBFGSwithL2(num_iterations=20).cost(n, d, k, sparsity, num_machines, cw, mw, nw),
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
        if isinstance(data, SparseMatrix):
            return self._fit_sparse(data, labels)
        ds = _as_dataset(self.ctx, data)
        lb = _as_dataset(ds.ctx, labels)
        n_total = ds.rows * max(1, ds.ctx.world_size)
        choice = self.optimize(n_total, ds.cols, lb.cols, 1.0, self.num_machines or ds.ctx.world_size)
        if choice == "exact":
            self.used = "exact"
            return LinearMapEstimator(self.lam, ds.ctx).fit(ds, lb)
        self.used = "block"
        return BlockLeastSquaresEstimator(1000, 3, self.lam, ctx=ds.ctx).fit(ds, lb)

    def _fit_sparse(self, sm: SparseMatrix, labels) -> BlockLinearMapper:
        lb = _as_dataset(sm.ctx, labels)
        n_total = sm.rows * max(1, sm.ctx.world_size)
        sparsity = sm.nnz / max(1, sm.rows * sm.cols)   # from the local shard, as n is
        choice = self.optimize(n_total, sm.cols, lb.cols, sparsity, self.num_machines or sm.ctx.world_size)
        if choice == "sparse_lbfgs":
            self.used = "sparse_lbfgs"
            return SparseLBFGSwithL2(num_iterations=20, reg_param=self.lam, ctx=sm.ctx).fit(sm, lb)
        dense = Densify().apply(sm)
        if choice == "exact":
            self.used = "exact"
            return LinearMapEstimator(self.lam, sm.ctx).fit(dense, lb)
        self.used = "block"
        return BlockLeastSquaresEstimator(1000, 3, self.lam, ctx=sm.ctx).fit(dense, lb)


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


# ------------------------------------------------------------------------------------------ PCA and ZCA whitening
class PCATransformer(LinearMapper):
    """``new PCATransformer(pcaMat)`` (K/nodes/learning/PCA.scala:19-31): x -> pcaMat^T x, a LinearMapper with no mean and no
    intercept (the reference does not centre).  ``pca_mat`` is d x dims."""

    @property
    def pca_mat(self) -> np.ndarray:
        return self.x

    @classmethod
    def from_matrix(cls, ctx: Context, pca_mat: np.ndarray) -> "PCATransformer":
        return cls.from_arrays(ctx, np.asarray(pca_mat, dtype=np.float64))


class BatchPCATransformer(Transformer):
    """``BatchPCATransformer(pcaMat)`` (PCA.scala:39-44): each (d x m_i) item -> pcaMat^T M_i (dims x m_i).  The columns of all items
    go through one device apply."""

    def __init__(self, transformer: PCATransformer):
        self.transformer = transformer

    @property
    def pca_mat(self) -> np.ndarray:
        return self.transformer.pca_mat

    def apply(self, data):
        if isinstance(data, ItemBatch):  # device items (LCSExtractor output): one apply over all rows, offsets kept
            if data.cols != self.pca_mat.shape[0]:
                raise ValueError(f"every item must have {self.pca_mat.shape[0]} rows")
            return ItemBatch(self.transformer.apply(data.matrix), data.offsets)
        single = isinstance(data, np.ndarray) and data.ndim == 2
        items = [np.asarray(data)] if single else [np.asarray(m) for m in data]
        d = self.pca_mat.shape[0]
        for m in items:
            if m.ndim != 2 or m.shape[0] != d:
                raise ValueError(f"every item must have {d} rows")
        rows = np.concatenate([m.T for m in items], 0).astype(np.float32)
        out = self.transformer.apply(self.transformer.ctx.matrix(rows)).to_numpy()
        offs = np.cumsum([0] + [m.shape[1] for m in items])
        res = [np.ascontiguousarray(out[offs[i]:offs[i + 1]].T) for i in range(len(items))]
        return res[0] if single else res


def _device_matrix(ctx: Optional[Context], data) -> DeviceMatrix:
    """A materialised device matrix of ``data`` (lazy feature sources are materialised first, as LinearMapEstimator.fit does)."""
    ds = _as_dataset(ctx, data)
    return ds if isinstance(ds, DeviceMatrix) else ds.materialize()


def _check_dims(dims) -> int:
    if int(dims) < 1:
        raise ValueError("dims must be >= 1")
    return int(dims)


class PCAEstimator(Estimator):
    """``new PCAEstimator(dims)`` (PCA.scala:157-225): the first ``dims`` eigenvectors of the exactly centred covariance, in
    descending order with the MATLAB sign convention.  The covariance is an fp64 DMMA Gram over the row shards and the eigenproblem
    is solved in fp64 (DESIGN.md section 15); after a fit ``eigenvalues`` holds the leading dims eigenvalues of X_c^T X_c."""

    def __init__(self, dims: int, ctx: Optional[Context] = None):
        self.dims, self.ctx = _check_dims(dims), ctx
        self.stats: Optional[dict] = None
        self.eigenvalues: Optional[np.ndarray] = None

    def fit(self, data) -> PCATransformer:
        """Collective with several ranks (data: this rank's rows)."""
        x = _device_matrix(self.ctx, data)
        h = C.c_int64(0)
        check(x.ctx.handle, lib().ks_pca_fit(x.ctx.handle, x.handle, self.dims, C.byref(h)))
        model = PCATransformer(x.ctx, h.value)
        self.stats = x.ctx.last_fit_stats()
        self.eigenvalues = np.asarray(self.stats["eigenvalues"], dtype=np.float64)
        return model

    def cost(self, n: int, d: int, k: int, sparsity: float, num_machines: int, cpu_weight: float, mem_weight: float,
             network_weight: float) -> float:
        """CostModel.cost (PCA.scala:211-224)."""
        flops = float(n) * d * d
        bytes_scanned = float(n) * d
        network = float(n) * d
        return max(cpu_weight * flops, mem_weight * bytes_scanned) + network_weight * network


class DistributedPCAEstimator(PCAEstimator):
    """``new DistributedPCAEstimator(dims)`` (K/nodes/learning/DistributedPCA.scala:20-74).  The reference's TSQR-then-SVD and the
    local SVD give the same components; on the device both are one algorithm, because the rows are sharded already."""

    def cost(self, n: int, d: int, k: int, sparsity: float, num_machines: int, cpu_weight: float, mem_weight: float,
             network_weight: float) -> float:
        """CostModel.cost (DistributedPCA.scala:59-73)."""
        log2m = math.log(num_machines) / math.log(2.0)
        flops = float(n) * d * d / num_machines + float(d) * d * d * log2m
        bytes_scanned = float(n) * d
        network = float(d) * d * log2m
        return max(cpu_weight * flops, mem_weight * bytes_scanned) + network_weight * network


def _columns_as_rows(data) -> np.ndarray:
    """The columns of every (d x m_i) item as rows (MatrixUtils.matrixToColArray)."""
    items = [np.asarray(data)] if isinstance(data, np.ndarray) and data.ndim == 2 else [np.asarray(m) for m in data]
    return np.concatenate([m.T for m in items], 0).astype(np.float32)


class LocalColumnPCAEstimator(Estimator):
    """``LocalColumnPCAEstimator(dims)`` (PCA.scala:51-72): PCA over the columns of (d x m_i) items -> BatchPCATransformer."""

    _inner = PCAEstimator

    def __init__(self, dims: int, ctx: Optional[Context] = None):
        self.dims, self.ctx = _check_dims(dims), ctx
        self.pca_estimator = self._inner(dims, ctx)

    def fit(self, data) -> BatchPCATransformer:
        if self.ctx is None:
            raise KeystoneError(-1, "numpy input needs a Context (pass ctx= to the node)")
        return BatchPCATransformer(self.pca_estimator.fit(self.ctx.matrix(_columns_as_rows(data))))

    def cost(self, n, d, k, sparsity, num_machines, cpu_weight, mem_weight, network_weight) -> float:
        return self.pca_estimator.cost(n, d, k, sparsity, num_machines, cpu_weight, mem_weight, network_weight)


class DistributedColumnPCAEstimator(LocalColumnPCAEstimator):
    """``DistributedColumnPCAEstimator(dims)`` (PCA.scala:81-102)."""

    _inner = DistributedPCAEstimator


class ColumnPCAEstimator(Estimator):
    """``ColumnPCAEstimator(dims, numMachines, cpuWeight, memWeight, networkWeight)`` (PCA.scala:117-151): ``optimize`` picks the
    local or the distributed column estimator by their costs (host-only arithmetic); ``fit`` uses the distributed one, the
    reference's default."""

    def __init__(self, dims: int, num_machines: Optional[int] = None, cpu_weight: float = 3.8e-4, mem_weight: float = 2.9e-1,
                 network_weight: float = 1.32, ctx: Optional[Context] = None):
        self.dims, self.num_machines, self.ctx = _check_dims(dims), num_machines, ctx
        self.cpu_weight, self.mem_weight, self.network_weight = cpu_weight, mem_weight, network_weight
        self.local_estimator = LocalColumnPCAEstimator(dims, ctx)
        self.distributed_estimator = DistributedColumnPCAEstimator(dims, ctx)
        self.default = self.distributed_estimator

    def optimize(self, sample: Sequence[np.ndarray], num_per_partition: dict) -> LocalColumnPCAEstimator:
        """sample: (d x m_i) items; num_per_partition: items per partition of the full dataset (WorkflowUtils.numPerPartition)."""
        cols_per_matrix = sum(np.asarray(m).shape[1] for m in sample) / float(len(sample))
        n = int(cols_per_matrix * sum(num_per_partition.values()))
        d = np.asarray(sample[0]).shape[0]
        m = self.num_machines or 1
        args = (n, d, self.dims, 1.0, m, self.cpu_weight, self.mem_weight, self.network_weight)
        local, dist = self.local_estimator.cost(*args), self.distributed_estimator.cost(*args)
        return self.local_estimator if local < dist else self.distributed_estimator

    def fit(self, data) -> BatchPCATransformer:
        return self.default.fit(data)


class ApproximatePCAEstimator(Estimator):
    """``new ApproximatePCAEstimator(dims, q, p)`` (K/nodes/learning/ApproximatePCA.scala:21-58; Halko, Martinsson and Tropp 2011,
    Algorithms 4.4 and 5.1) on the raw, uncentred data.  The Gaussian test matrix Omega (d x (dims + p)) is drawn on the host by
    ``ApproximatePCAEstimator.omega``: ``numpy.random.default_rng(seed).standard_normal``.  Breeze's MersenneTwister stream is not
    reproduced.  The QR of every tall-skinny factor is shifted CholeskyQR3 in fp64 (DESIGN.md section 15)."""

    def __init__(self, dims: int, q: int = 10, p: int = 5, seed: int = 0, ctx: Optional[Context] = None):
        if int(q) < 0:
            raise ValueError("q must be >= 0")
        if int(p) < 0:
            raise ValueError("p must be >= 0")
        self.dims, self.q, self.p, self.seed, self.ctx = _check_dims(dims), int(q), int(p), seed, ctx
        self.stats: Optional[dict] = None
        self.singular_values: Optional[np.ndarray] = None

    @staticmethod
    def omega(d: int, l: int, seed: int = 0) -> np.ndarray:
        """The d x l Gaussian test matrix of a fit with this seed."""
        return np.random.default_rng(seed).standard_normal((int(d), int(l)))

    def fit(self, data) -> PCATransformer:
        """Collective with several ranks (data: this rank's rows; every rank draws the same Omega)."""
        x = _device_matrix(self.ctx, data)
        om = np.asfortranarray(self.omega(x.cols, self.dims + self.p, self.seed))
        h = C.c_int64(0)
        check(x.ctx.handle, lib().ks_approx_pca_fit(x.ctx.handle, x.handle, om.ctypes.data_as(C.c_void_p), self.dims, self.q, self.p,
                                                     C.byref(h)))
        model = PCATransformer(x.ctx, h.value)
        self.stats = x.ctx.last_fit_stats()
        self.singular_values = np.asarray(self.stats["singular_values"], dtype=np.float64)
        return model

    @staticmethod
    def approximate_q(data, l: int, q: int, seed: int = 0, ctx: Optional[Context] = None) -> DeviceMatrix:
        """``ApproximatePCAEstimator.approximateQ(A, l, q, seed)`` (ApproximatePCA.scala:69-85): this rank's rows of the orthonormal
        N x l basis, as an fp32 device matrix."""
        x = _device_matrix(ctx, data)
        om = np.asfortranarray(ApproximatePCAEstimator.omega(x.cols, l, seed))
        h = C.c_int64(0)
        check(x.ctx.handle, lib().ks_approx_range(x.ctx.handle, x.handle, om.ctypes.data_as(C.c_void_p), int(l), int(q), C.byref(h)))
        return DeviceMatrix(x.ctx, h.value, x.rows, int(l))


class ZCAWhitener(LinearMapper):
    """``new ZCAWhitener(whitener, means)`` (K/nodes/learning/ZCAWhitener.scala:12-19): (in - means) * whitener, a LinearMapper
    with the means as its feature scaler."""

    @property
    def whitener(self) -> np.ndarray:
        return self.x

    @property
    def means(self) -> np.ndarray:
        return self.feature_means[0]

    @classmethod
    def from_whitener(cls, ctx: Context, whitener: np.ndarray, means: np.ndarray) -> "ZCAWhitener":
        return cls.from_arrays(ctx, np.asarray(whitener, dtype=np.float64), None, np.asarray(means, dtype=np.float64))


class ZCAWhitenerEstimator(Estimator):
    """``new ZCAWhitenerEstimator(eps)`` (ZCAWhitener.scala:30-72): whitener = V diag((lambda / (N - 1) + eps)^-1/2) V^T from the
    eigenpairs of the exactly centred covariance, all in fp64 on the device (DESIGN.md section 15).  Needs at least d rows."""

    def __init__(self, eps: float = 0.1, ctx: Optional[Context] = None):
        eps = float(eps)
        if not (eps >= 0.0 and math.isfinite(eps)):
            raise ValueError("eps must be finite and >= 0")
        self.eps, self.ctx = eps, ctx
        self.stats: Optional[dict] = None

    def fit_single(self, matrix) -> ZCAWhitener:
        """Collective with several ranks (matrix: this rank's rows)."""
        x = _device_matrix(self.ctx, matrix)
        h = C.c_int64(0)
        check(x.ctx.handle, lib().ks_zca_fit(x.ctx.handle, x.handle, self.eps, C.byref(h)))
        model = ZCAWhitener(x.ctx, h.value)
        self.stats = x.ctx.last_fit_stats()
        return model

    def fit(self, data) -> ZCAWhitener:
        """Fits on the first item of a sequence of matrices (ZCAWhitener.scala:33-35); a single matrix is its own first item."""
        if isinstance(data, (list, tuple)):
            data = data[0]
        return self.fit_single(data)


class StandardScalerModel(Transformer):
    """``StandardScalerModel(mean, std)`` (K/nodes/stats/StandardScaler.scala:16-31): (x - mean) [/ std], computed on the device in
    fp64 and rounded once to fp32 (``ks_standard_scaler_apply``).  ``std=None`` only centres."""

    def __init__(self, mean: np.ndarray, std: Optional[np.ndarray] = None, ctx: Optional[Context] = None):
        self.mean, self.std, self.ctx = mean, std, ctx

    def apply(self, data) -> DeviceMatrix:
        x = _device_matrix(self.ctx, data)
        mean = np.ascontiguousarray(self.mean, dtype=np.float64).reshape(-1)
        std = None if self.std is None else np.ascontiguousarray(self.std, dtype=np.float64).reshape(-1)
        if mean.size != x.cols or (std is not None and std.size != x.cols):
            raise ValueError("StandardScalerModel: mean and std need one value per column")
        h = C.c_int64(0)
        check(x.ctx.handle, lib().ks_standard_scaler_apply(x.ctx.handle, x.handle, mean.ctypes.data_as(C.c_void_p),
                                                           None if std is None else std.ctypes.data_as(C.c_void_p), C.byref(h)))
        return DeviceMatrix(x.ctx, h.value, x.rows, x.cols)


class StandardScaler(Estimator):
    """``new StandardScaler(normalizeStdDev, eps)`` (StandardScaler.scala:38-59): fp64 column means and, with ``normalizeStdDev``, the
    unbiased column std (MLlib's ``MultivariateOnlineSummarizer``), 1.0 where the std is NaN, infinite or below ``eps``.  The sums run
    in a fixed order, so a refit is bit-identical.  Collective with several ranks (data: this rank's rows)."""

    def __init__(self, normalizeStdDev: bool = True, eps: float = 1e-12, ctx: Optional[Context] = None):
        self.normalize_std, self.eps, self.ctx = bool(normalizeStdDev), float(eps), ctx

    def fit(self, data) -> StandardScalerModel:
        x = _device_matrix(self.ctx, data)
        mean = np.empty(x.cols, dtype=np.float64)
        std = np.empty(x.cols, dtype=np.float64)
        check(x.ctx.handle, lib().ks_standard_scaler_fit(x.ctx.handle, x.handle, 1 if self.normalize_std else 0, self.eps,
                                                         mean.ctypes.data_as(C.c_void_p), std.ctypes.data_as(C.c_void_p)))
        return StandardScalerModel(mean, std if self.normalize_std else None, x.ctx)


def stats_normalize_rows(data, alpha: float = 1.0, ctx: Optional[Context] = None) -> DeviceMatrix:
    """``Stats.normalizeRows(mat, alpha)`` (K/utils/Stats.scala:112-123) on the device: per row, minus the mean, over
    sqrt(sample variance + alpha), in fp64, rounded once to fp32."""
    x = _device_matrix(ctx, data)
    h = C.c_int64(0)
    check(x.ctx.handle, lib().ks_matrix_stats_normalize_rows(x.ctx.handle, x.handle, float(alpha), C.byref(h)))
    return DeviceMatrix(x.ctx, h.value, x.rows, x.cols)


# ------------------------------------------------------------------------------------------ LCS Fisher-vector branch
# LCSExtractor -> BatchPCATransformer -> FisherVector(gmm) -> FloatToDouble -> MatrixVectorizer -> NormalizeRows -> SignedHellingerMapper
# -> NormalizeRows (K/pipelines/images/imagenet/ImageNetSiftLcsFV.scala).  DESIGN.md section 16.
class ItemBatch(Dataset):
    """A batch of items -- the reference's one (dim x n_i) ``DenseMatrix[Float]`` per image -- as ONE device matrix holding the columns
    of every item as rows, plus item row offsets: item i is rows [offsets[i], offsets[i + 1])."""

    def __init__(self, matrix: DeviceMatrix, offsets):
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        if offsets.ndim != 1 or offsets.size < 1 or offsets[0] != 0 or offsets[-1] != matrix.rows or (np.diff(offsets) < 0).any():
            raise ValueError("item offsets must start at 0, end at the row count and never decrease")
        self.ctx, self.matrix, self.offsets = matrix.ctx, matrix, offsets

    @classmethod
    def from_items(cls, ctx: Context, items: Sequence[np.ndarray]) -> "ItemBatch":
        """Uploads (dim x n_i) host matrices."""
        items = [np.atleast_2d(np.asarray(m)) for m in items]
        offsets = np.cumsum([0] + [m.shape[1] for m in items])
        return cls(ctx.matrix(np.concatenate([m.T for m in items], 0).astype(np.float32)), offsets)

    @property
    def n_items(self) -> int:
        return int(self.offsets.size - 1)

    @property
    def rows(self) -> int:
        return self.matrix.rows

    @property
    def cols(self) -> int:
        return self.matrix.cols

    def to_list(self, dtype=np.float64) -> List[np.ndarray]:
        """The items as the reference's (dim x n_i) matrices."""
        host = self.matrix.to_numpy(dtype)
        return [np.ascontiguousarray(host[self.offsets[i]:self.offsets[i + 1]].T) for i in range(self.n_items)]

    def to_numpy(self, dtype=np.float64) -> np.ndarray:
        return self.matrix.to_numpy(dtype)


class ImageBatch(Dataset):
    """Equal-size images as rows of a device matrix in ImageVectorizer order (value (x, y, c) at c + x*C + y*C*xDim, x = row)."""

    def __init__(self, matrix: DeviceMatrix, x_dim: int, y_dim: int, channels: int):
        if matrix.cols != x_dim * y_dim * channels:
            raise ValueError("image matrix columns must equal x_dim * y_dim * channels")
        self.ctx, self.matrix = matrix.ctx, matrix
        self.x_dim, self.y_dim, self.channels = int(x_dim), int(y_dim), int(channels)

    @classmethod
    def from_images(cls, ctx: Context, images_xyc: np.ndarray) -> "ImageBatch":
        """(n, x, y, c) host images."""
        a = np.asarray(images_xyc)
        return cls(ctx.matrix(images_to_matrix(a)), a.shape[1], a.shape[2], a.shape[3])

    @property
    def rows(self) -> int:
        return self.matrix.rows


class LCSExtractor(Transformer):
    """``new LCSExtractor(stride, strideStart, subPatchSize)`` (K/nodes/images/LCSExtractor.scala): per keypoint, the mean and standard
    deviation of every channel over n x n neighbouring s x s windows (96 values for 3 channels and the defaults).  Window statistics in
    fp64, rounded once to fp32.  Input: an ``ImageBatch``, an (n, x, y, c) array, one (x, y, c) image (returns its (dim x nKP) matrix)
    or a list of images, grouped by shape.  Output: an ``ItemBatch`` with one item per image."""

    def __init__(self, stride: int, strideStart: int, subPatchSize: int, ctx: Optional[Context] = None):
        self.stride, self.stride_start, self.sub_patch_size, self.ctx = int(stride), int(strideStart), int(subPatchSize), ctx

    def keypoints(self, x_dim: int, y_dim: int) -> int:
        return len(range(self.stride_start, x_dim - self.stride_start, self.stride)) * \
            len(range(self.stride_start, y_dim - self.stride_start, self.stride))

    def _extract(self, batch: ImageBatch) -> ItemBatch:
        h = C.c_int64(0)
        check(batch.ctx.handle, lib().ks_lcs_extract(batch.ctx.handle, batch.matrix.handle, batch.x_dim, batch.y_dim, batch.channels,
                                                      self.stride, self.stride_start, self.sub_patch_size, C.byref(h)))
        rows, cols = C.c_int64(0), C.c_int64(0)
        check(batch.ctx.handle, lib().ks_matrix_shape(batch.ctx.handle, h.value, C.byref(rows), C.byref(cols)))
        nkp = self.keypoints(batch.x_dim, batch.y_dim)
        return ItemBatch(DeviceMatrix(batch.ctx, h.value, rows.value, cols.value), np.arange(batch.rows + 1, dtype=np.int64) * nkp)

    def apply(self, data):
        if isinstance(data, ImageBatch):
            return self._extract(data)
        if self.ctx is None:
            raise KeystoneError(-1, "numpy input needs a Context (pass ctx= to the node)")
        if isinstance(data, np.ndarray) and data.ndim == 3:
            return self._extract(ImageBatch.from_images(self.ctx, data[None])).to_list(np.float32)[0]
        if isinstance(data, np.ndarray) and data.ndim == 4:
            return self._extract(ImageBatch.from_images(self.ctx, data))
        images = [np.asarray(im) for im in data]
        groups = {}
        for i, im in enumerate(images):
            groups.setdefault(im.shape, []).append(i)
        if len(groups) == 1:
            return self._extract(ImageBatch.from_images(self.ctx, np.stack(images)))
        # several shapes: one launch per shape, the items put back in input order on the host
        items: List[Optional[np.ndarray]] = [None] * len(images)
        for idx in groups.values():
            for i, m in zip(idx, self._extract(ImageBatch.from_images(self.ctx, np.stack([images[i] for i in idx]))).to_list(np.float32)):
                items[i] = m
        return ItemBatch.from_items(self.ctx, items)


class _GmmHandle:
    def __init__(self, ctx: Context, handle: int):
        self.ctx, self.handle = ctx, handle

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                lib().ks_gmm_destroy(self.ctx.handle, self.handle)
        except Exception:
            pass


class GaussianMixtureModel(Transformer):
    """``GaussianMixtureModel(means, variances, weights, weightThreshold)`` (K/nodes/learning/GaussianMixtureModel.scala): means and
    variances are dim x k (one column per component).  ``apply`` returns the thresholded posteriors, computed in fp64 on the device:
    a vector for a vector, a device batch (N x k) for a batch.  The device copy is made per Context, on first use or when ``ctx`` is
    given."""

    def __init__(self, means, variances, weights, weightThreshold: float = 1e-4, ctx: Optional[Context] = None):
        self.means = np.asarray(means, dtype=np.float64)
        self.variances = np.asarray(variances, dtype=np.float64)
        self.weights = np.asarray(weights, dtype=np.float64).reshape(-1)
        if self.means.ndim != 2 or self.means.shape != self.variances.shape:
            raise ValueError("GMM means and variances must be the same size.")
        if self.weights.size != self.means.shape[1]:
            raise ValueError("Every GMM center must have a weight.")
        self.weight_threshold, self.ctx = float(weightThreshold), ctx
        self._handles = {}
        if ctx is not None:
            self.handle(ctx)

    @property
    def dim(self) -> int:
        return self.means.shape[0]

    @property
    def k(self) -> int:
        return self.means.shape[1]

    @classmethod
    def load(cls, meanFile: str, varsFile: str, weightsFile: str, ctx: Optional[Context] = None) -> "GaussianMixtureModel":
        """``GaussianMixtureModel.load`` (GaussianMixtureModel.scala:95-105): headerless CSVs, means and variances dim x k; the weights
        file flattened column-major (csvread(...).toDenseVector)."""
        from .loaders import CsvDataLoader
        w = CsvDataLoader(weightsFile, np.float64).reshape(-1, order="F")
        return cls(CsvDataLoader(meanFile, np.float64), CsvDataLoader(varsFile, np.float64), w, ctx=ctx)

    def handle(self, ctx: Context) -> int:
        owner = self._handles.get(ctx.handle)
        if owner is None:
            m, v = np.asfortranarray(self.means), np.asfortranarray(self.variances)
            w = np.ascontiguousarray(self.weights)
            h = C.c_int64(0)
            check(ctx.handle, lib().ks_gmm_create(ctx.handle, m.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p),
                                                   w.ctypes.data_as(C.c_void_p), self.dim, self.k, self.weight_threshold, C.byref(h)))
            owner = self._handles[ctx.handle] = _GmmHandle(ctx, h.value)
        return owner.handle

    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 1
        x = _device_matrix(self.ctx, data)
        h = C.c_int64(0)
        check(x.ctx.handle, lib().ks_gmm_posteriors(x.ctx.handle, self.handle(x.ctx), x.handle, C.byref(h)))
        out = DeviceMatrix(x.ctx, h.value, x.rows, self.k)
        return out.to_numpy()[0] if single else out


class FisherVector(Transformer):
    """``FisherVector(gmm)`` (K/nodes/images/FisherVector.scala) followed by MatrixVectorizer: one row of 2 dim k values per item,
    element (d, j) of the reference's dim x 2k matrix [fv1 | fv2] at column d + dim * j.  Posteriors and statistics stay on the
    device in fp64; the output is fp32.  fv2 follows Sanchez et al. (DESIGN.md section 16).  Input: an ``ItemBatch``, a list of
    (dim x n_i) matrices, or one such matrix (returns its dim x 2k matrix)."""

    def __init__(self, gmm: GaussianMixtureModel):
        self.gmm = gmm

    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 2
        if not isinstance(data, ItemBatch):
            ctx = self.gmm.ctx
            if ctx is None:
                raise KeystoneError(-1, "host items need a Context (pass ctx= to the GaussianMixtureModel)")
            data = ItemBatch.from_items(ctx, [data] if single else list(data))
        ctx = data.ctx
        offs = data.offsets
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_fisher_vector_apply(ctx.handle, self.gmm.handle(ctx), data.matrix.handle, offs.ctypes.data_as(C.c_void_p),
                                                        data.n_items, C.byref(h)))
        out = DeviceMatrix(ctx, h.value, data.n_items, 2 * self.gmm.dim * self.gmm.k)
        if single:
            return out.to_numpy()[0].reshape(2 * self.gmm.k, self.gmm.dim).T.copy()
        return out


class FloatToDouble(Transformer):
    """K/nodes/util/FloatToDouble: device storage is fp32 and every consumer computes in fp64, so this passes its input through."""

    def apply(self, data):
        return data


class MatrixVectorizer(Transformer):
    """K/nodes/util/MatrixVectorizer: ``FisherVector`` already writes each item's matrix column-major as one row, so this passes its
    input through."""

    def apply(self, data):
        return data


def _map_rows(data, ctx: Optional[Context], fn) -> object:
    """Applies a device row map to a batch (DeviceMatrix, ItemBatch: offsets kept) or a host vector / matrix."""
    if isinstance(data, ItemBatch):
        return ItemBatch(fn(data.matrix), data.offsets)
    single = isinstance(data, np.ndarray) and data.ndim == 1
    out = fn(_device_matrix(ctx, data))
    return out.to_numpy()[0] if single else out


def _normalize_rows(x: DeviceMatrix) -> DeviceMatrix:
    h = C.c_int64(0)
    check(x.ctx.handle, lib().ks_matrix_normalize_rows(x.ctx.handle, x.handle, C.byref(h)))
    return DeviceMatrix(x.ctx, h.value, x.rows, x.cols)


def _signed_sqrt(x: DeviceMatrix) -> DeviceMatrix:
    h = C.c_int64(0)
    check(x.ctx.handle, lib().ks_matrix_map(x.ctx.handle, x.handle, 2, None, 0.0, 0.0, C.byref(h)))
    return DeviceMatrix(x.ctx, h.value, x.rows, x.cols)


class NormalizeRows(Transformer):
    """NormalizeRows (K/nodes/stats/NormalizeRows.scala): each row divided by max(|row|_2, 2.2e-16), the norm in fp64."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    def apply(self, data):
        return _map_rows(data, self.ctx, _normalize_rows)


class SignedHellingerMapper(Transformer):
    """SignedHellingerMapper (K/nodes/stats/SignedHellingerMapper.scala): sign(v) sqrt(|v|) elementwise."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    def apply(self, data):
        return _map_rows(data, self.ctx, _signed_sqrt)


class BatchSignedHellingerMapper(SignedHellingerMapper):
    """BatchSignedHellingerMapper: the same map on (dim x n) Float items (an ``ItemBatch`` keeps its offsets)."""


# ------------------------------------------------------------------------------------------ mixture and k-means fits
# GaussianMixtureModelEstimator, KMeansPlusPlusEstimator / KMeansModel, (Scala)GMMFisherVectorEstimator, ColumnSampler
# (K/nodes/learning/{GaussianMixtureModelEstimator,KMeansPlusPlus}.scala, K/nodes/images/FisherVector.scala:55-95,
# K/nodes/stats/Sampling.scala).  DESIGN.md section 17.
def _fit_rows(ctx: Optional[Context], data) -> DeviceMatrix:
    """The sample rows of a fit: an ``ItemBatch`` (every descriptor is a sample), a device matrix or host rows."""
    if isinstance(data, ItemBatch):
        return data.matrix
    return _device_matrix(ctx, data)


class KMeansModel(Transformer):
    """``KMeansModel(means)`` (KMeansPlusPlus.scala:16-70), means numMeans x dim: ``apply`` returns the one-hot assignment to the first
    nearest mean (a vector for a vector, an N x numMeans device batch for a batch)."""

    def __init__(self, means, ctx: Optional[Context] = None):
        self.means = np.ascontiguousarray(np.atleast_2d(np.asarray(means, dtype=np.float64)))
        self.ctx = ctx

    def apply(self, data):
        single = isinstance(data, np.ndarray) and data.ndim == 1
        x = _device_matrix(self.ctx, data)
        h = C.c_int64(0)
        k, d = self.means.shape
        check(x.ctx.handle, lib().ks_kmeans_assign(x.ctx.handle, x.handle, self.means.ctypes.data_as(C.c_void_p), k, d, C.byref(h)))
        out = DeviceMatrix(x.ctx, h.value, x.rows, k)
        return out.to_numpy()[0] if single else out


class KMeansPlusPlusEstimator(Estimator):
    """``KMeansPlusPlusEstimator(numMeans, maxIterations, stopTolerance, seed)`` (KMeansPlusPlus.scala:83-181): k-means++ seeding and
    Lloyd passes on the device in fp64.  The seeding draws take ``numMeans`` uniforms from ``numpy.random.default_rng(seed)``, with the
    draw rule of include/keystone_b200.h; Breeze's MersenneTwister stream is not reproduced.  After a fit ``seed_rows`` holds the
    seed rows and ``stats`` the fit's statistics (cost history, stop reason, per-phase times)."""

    def __init__(self, numMeans: int, maxIterations: int, stopTolerance: float = 1e-3, seed: int = 0, ctx: Optional[Context] = None):
        self.num_means, self.max_iterations, self.stop_tolerance = int(numMeans), int(maxIterations), float(stopTolerance)
        self.seed, self.ctx = seed, ctx
        self.seed_rows: Optional[np.ndarray] = None
        self.stats: Optional[dict] = None

    def uniforms(self) -> np.ndarray:
        return np.random.default_rng(self.seed).random(self.num_means)

    def fit(self, data) -> KMeansModel:
        x = _fit_rows(self.ctx, data)
        u = self.uniforms()
        means = np.zeros((self.num_means, x.cols))
        seeds = np.zeros(self.num_means, dtype=np.int64)
        it = C.c_int32(0)
        check(x.ctx.handle, lib().ks_kmeans_fit(x.ctx.handle, x.handle, self.num_means, self.max_iterations, self.stop_tolerance,
                                                 u.ctypes.data_as(C.c_void_p), means.ctypes.data_as(C.c_void_p),
                                                 seeds.ctypes.data_as(C.c_void_p), C.byref(it)))
        self.seed_rows, self.stats = seeds, x.ctx.last_fit_stats()
        return KMeansModel(means, x.ctx)


KMEANS_PLUS_PLUS_INITIALIZATION = "KMEANS_PLUS_PLUS_INITIALIZATION"
RANDOM_INITIALIZATION = "RANDOM_INITIALIZATION"


class GaussianMixtureModelEstimator(Estimator):
    """``GaussianMixtureModelEstimator(k, maxIterations, minClusterSize, stopTolerance, weightThreshold, smallVarianceThreshold,
    absoluteVarianceThreshold, initializationMethod, seed)`` (GaussianMixtureModelEstimator.scala): diagonal-covariance EM in fp64 on
    the device, started from k-means++ (one Lloyd pass) or from random means.  The uniforms come from
    ``numpy.random.default_rng(seed)`` (k of them for k-means++, k x dim for the random start); Breeze's stream is not reproduced.
    The fitted ``GaussianMixtureModel`` carries the default weightThreshold 1e-4, as the reference's does, and already holds its
    device copy for the fit's Context.  After a fit ``stats`` holds the iterations, stop reason and cost history."""

    def __init__(self, k: int, maxIterations: int = 100, minClusterSize: int = 40, stopTolerance: float = 1e-4,
                 weightThreshold: float = 1e-4, smallVarianceThreshold: float = 1e-2, absoluteVarianceThreshold: float = 1e-9,
                 initializationMethod: str = KMEANS_PLUS_PLUS_INITIALIZATION, seed: int = 0, ctx: Optional[Context] = None):
        if int(minClusterSize) <= 0:
            raise ValueError("Minimum cluster size must be positive")
        if int(maxIterations) <= 0:
            raise ValueError("maxIterations must be positive")
        if initializationMethod not in (KMEANS_PLUS_PLUS_INITIALIZATION, RANDOM_INITIALIZATION):
            raise ValueError("initializationMethod must be KMEANS_PLUS_PLUS_INITIALIZATION or RANDOM_INITIALIZATION")
        self.k, self.max_iterations, self.min_cluster_size = int(k), int(maxIterations), int(minClusterSize)
        self.stop_tolerance, self.weight_threshold = float(stopTolerance), float(weightThreshold)
        self.small_variance_threshold, self.absolute_variance_threshold = float(smallVarianceThreshold), float(absoluteVarianceThreshold)
        self.initialization_method, self.seed, self.ctx = initializationMethod, seed, ctx
        self.stats: Optional[dict] = None

    def uniforms(self, dim: int) -> np.ndarray:
        rng = np.random.default_rng(self.seed)
        return rng.random(self.k) if self.initialization_method == KMEANS_PLUS_PLUS_INITIALIZATION else rng.random((self.k, int(dim)))

    def fit(self, data) -> GaussianMixtureModel:
        x = _fit_rows(self.ctx, data)
        u = np.ascontiguousarray(self.uniforms(x.cols))
        means, variances = np.zeros((x.cols, self.k), order="F"), np.zeros((x.cols, self.k), order="F")
        weights = np.zeros(self.k)
        h, it = C.c_int64(0), C.c_int32(0)
        init = 0 if self.initialization_method == KMEANS_PLUS_PLUS_INITIALIZATION else 1
        check(x.ctx.handle, lib().ks_gmm_fit(x.ctx.handle, x.handle, self.k, self.max_iterations, float(self.min_cluster_size),
                                              self.stop_tolerance, self.weight_threshold, self.small_variance_threshold,
                                              self.absolute_variance_threshold, init, u.ctypes.data_as(C.c_void_p), C.byref(h),
                                              means.ctypes.data_as(C.c_void_p), variances.ctypes.data_as(C.c_void_p),
                                              weights.ctypes.data_as(C.c_void_p), C.byref(it)))
        owner = _GmmHandle(x.ctx, h.value)
        self.stats = x.ctx.last_fit_stats()
        gmm = GaussianMixtureModel(np.ascontiguousarray(means), np.ascontiguousarray(variances), weights)
        gmm.ctx = x.ctx
        gmm._handles[x.ctx.handle] = owner
        return gmm


class ScalaGMMFisherVectorEstimator(Estimator):
    """``ScalaGMMFisherVectorEstimator(k)`` (FisherVector.scala:55-72): fits ``GaussianMixtureModelEstimator(k)`` with its defaults
    on every descriptor of the items (an ``ItemBatch``'s rows, or the columns of (dim x n_i) matrices) and returns
    ``FisherVector(gmm)``."""

    def __init__(self, k: int, ctx: Optional[Context] = None):
        self.k, self.ctx = int(k), ctx
        self.gmm_estimator = GaussianMixtureModelEstimator(self.k, ctx=ctx)

    def fit(self, data) -> FisherVector:
        if not isinstance(data, ItemBatch):
            if self.ctx is None:
                raise KeystoneError(-1, "host items need a Context (pass ctx= to the estimator)")
            data = ItemBatch.from_items(self.ctx, [data] if isinstance(data, np.ndarray) and data.ndim == 2 else list(data))
        return FisherVector(self.gmm_estimator.fit(data))


class GMMFisherVectorEstimator(ScalaGMMFisherVectorEstimator):
    """``GMMFisherVectorEstimator(k)`` (FisherVector.scala:74-95).  The reference's optimizer switches to the EncEval C++ estimator
    for k >= 32; that is a different algorithm and is not provided, so this always takes the Scala path (the device EM)."""


class ColumnSampler(Transformer):
    """``ColumnSampler(numSamplesPerMatrix)`` (K/nodes/stats/Sampling.scala:12-21): per item, ``numSamplesPerMatrix`` columns drawn
    uniformly with replacement, gathered on the device into a new ``ItemBatch``.  Indices come from
    ``numpy.random.default_rng(seed)`` (``seed=None``: fresh entropy, as the reference's unseeded ``scala.util.Random``)."""

    def __init__(self, numSamplesPerMatrix: int, seed: Optional[int] = None, ctx: Optional[Context] = None):
        if int(numSamplesPerMatrix) < 0:
            raise ValueError("numSamplesPerMatrix must be >= 0")
        self.num_samples, self.seed, self.ctx = int(numSamplesPerMatrix), seed, ctx
        self._rng = np.random.default_rng(seed)

    def sample_rows(self, offsets: np.ndarray) -> np.ndarray:
        """The gathered rows of an item batch with these offsets (the next draws of this sampler's generator)."""
        sizes = np.diff(np.asarray(offsets, dtype=np.int64))
        if (sizes <= 0).any() and self.num_samples > 0:
            raise ValueError("ColumnSampler: every item needs at least one column")
        return np.concatenate([o + self._rng.integers(0, n, size=self.num_samples) for o, n in zip(offsets[:-1], sizes)]
                              + [np.zeros(0, dtype=np.int64)]).astype(np.int64)

    def apply(self, data):
        if not isinstance(data, ItemBatch):
            if self.ctx is None:
                raise KeystoneError(-1, "host items need a Context (pass ctx= to the node)")
            data = ItemBatch.from_items(self.ctx, list(data))
        rows = np.ascontiguousarray(self.sample_rows(data.offsets))
        h = C.c_int64(0)
        check(data.ctx.handle, lib().ks_matrix_gather_rows(data.ctx.handle, data.matrix.handle, rows.ctypes.data_as(C.c_void_p), rows.size,
                                                           C.byref(h)))
        out = DeviceMatrix(data.ctx, h.value, rows.size, data.cols)
        return ItemBatch(out, np.arange(data.n_items + 1, dtype=np.int64) * self.num_samples)


# ------------------------------------------------------------------------------------------------- dense SIFT branch
# PixelScaler -> GrayScaler -> SIFTExtractor, the head of K/pipelines/images/voc/VOCSIFTFisher.scala:41-44 and of the SIFT half of
# K/pipelines/images/imagenet/ImageNetSiftLcsFV.scala:99-101.  DESIGN.md section 18.
def _new_matrix(ctx: Context, handle: int) -> DeviceMatrix:
    rows, cols = C.c_int64(0), C.c_int64(0)
    check(ctx.handle, lib().ks_matrix_shape(ctx.handle, handle, C.byref(rows), C.byref(cols)))
    return DeviceMatrix(ctx, handle, rows.value, cols.value)


class _PixelScaledImages(ImageBatch):
    """PixelScaler's output: the source batch with x / 255.0 pending, so that GrayScaler can take it in fp64 together with the gray
    weights (the reference never rounds in between).  Reading ``matrix`` materialises the scaled values, rounded once to fp32."""

    def __init__(self, source: ImageBatch):
        self.ctx, self.source = source.ctx, source
        self.x_dim, self.y_dim, self.channels = source.x_dim, source.y_dim, source.channels
        self._matrix: Optional[DeviceMatrix] = None

    @property
    def matrix(self) -> DeviceMatrix:
        if self._matrix is None:
            h = C.c_int64(0)
            check(self.ctx.handle, lib().ks_image_pixel_scale(self.ctx.handle, self.source.matrix.handle, C.byref(h)))
            self._matrix = _new_matrix(self.ctx, h.value)
        return self._matrix

    @property
    def rows(self) -> int:
        return self.source.rows


def _image_batches(node, data):
    """Image inputs as (batches, restore): an ImageBatch, an (n, x, y, c) array, one (x, y, c) or (x, y) image, or a list of images and
    batches (one batch per shape); restore(per-batch results) puts per-image results back in input order."""
    def upload(a):
        if node.ctx is None:
            raise KeystoneError(-1, "numpy input needs a Context (pass ctx= to the node)")
        return ImageBatch.from_images(node.ctx, a)

    if isinstance(data, ImageBatch):
        return [data], None
    if isinstance(data, np.ndarray) and data.ndim == 4:
        return [upload(data)], None
    if isinstance(data, np.ndarray) and data.ndim in (2, 3):
        a = data if data.ndim == 3 else data[:, :, None]
        return [upload(a[None])], "single"
    items = list(data)
    groups = {}
    for i, im in enumerate(items):
        key = ("batch", i) if isinstance(im, ImageBatch) else np.asarray(im).shape
        groups.setdefault(key, []).append(i)
    batches, order = [], []
    for key, idx in groups.items():
        if key[0] == "batch":
            batches.append(items[idx[0]])
        else:
            ims = [np.asarray(items[i]) for i in idx]
            batches.append(upload(np.stack([m if m.ndim == 3 else m[:, :, None] for m in ims])))
        order.append(idx)
    return batches, order


def _per_batch(node, data, fn):
    """fn on an ImageBatch, on an array uploaded as one, or on each image of a list (a list of one-image batches, input order)."""
    if isinstance(data, (list, tuple)):
        return [fn(b if isinstance(b, ImageBatch) else _image_batches(node, np.asarray(b))[0][0]) for b in data]
    return fn(_image_batches(node, data)[0][0])


class PixelScaler(Transformer):
    """``PixelScaler`` (K/nodes/images/PixelScaler.scala): every value / 255.0, in fp64.  ImageBatch -> ImageBatch; the division is
    deferred so that a following GrayScaler computes both in fp64 and rounds once."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    def apply(self, data):
        return _per_batch(self, data, _PixelScaledImages)


class GrayScaler(Transformer):
    """``GrayScaler`` (K/nodes/images/GrayScaler.scala, ImageUtils.toGrayScale): 0.2989 R + 0.5870 G + 0.1140 B with the channels in
    BGR order for three channels, sqrt(mean of squares) otherwise, in fp64 (after PixelScaler's division when one precedes it),
    rounded once to fp32.  ImageBatch -> one-channel ImageBatch."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    @staticmethod
    def _gray(batch: ImageBatch) -> ImageBatch:
        scaled = isinstance(batch, _PixelScaledImages) and batch._matrix is None
        src = batch.source if scaled else batch
        h = C.c_int64(0)
        check(batch.ctx.handle, lib().ks_image_grayscale(batch.ctx.handle, src.matrix.handle, batch.x_dim, batch.y_dim, batch.channels,
                                                         1 if scaled else 0, C.byref(h)))
        return ImageBatch(_new_matrix(batch.ctx, h.value), batch.x_dim, batch.y_dim, 1)

    def apply(self, data):
        return _per_batch(self, data, self._gray)


class SIFTExtractor(Transformer):
    """``SIFTExtractor(stepSize, binSize, scales, scaleStep)`` (K/nodes/images/external/SIFTExtractor.scala): vlfeat's dense SIFT with a
    flat window at ``scales`` scales (bin ``binSize + 2s``, step ``stepSize + s scaleStep``), 128 integer values in [0, 255] per
    keypoint, zero below the contrast threshold.  Input: one-channel images -- an ``ImageBatch``, an (n, x, y, 1) array, one (x, y[, 1])
    image (returns its (128 x nKP) matrix, as the reference) or a list of images, grouped by shape, input order kept.  Output: an
    ``ItemBatch`` with one item per image, one descriptor per row."""

    descriptorSize = 128

    def __init__(self, stepSize: int = 3, binSize: int = 4, scales: int = 4, scaleStep: int = 1, ctx: Optional[Context] = None):
        self.step, self.bin, self.scales, self.scale_step, self.ctx = int(stepSize), int(binSize), int(scales), int(scaleStep), ctx

    def keypoints_per_scale(self, x_dim: int, y_dim: int) -> List[int]:
        counts = np.zeros(max(self.scales, 1), dtype=np.int64)
        rc = lib().ks_sift_keypoints(x_dim, y_dim, self.step, self.bin, self.scales, self.scale_step, counts.ctypes.data_as(_capi.p_i64))
        if rc != 0:
            raise KeystoneError(rc, "SIFTExtractor: invalid image shape or parameters (stepSize, binSize, scales >= 1, scaleStep >= 0)")
        return [int(v) for v in counts[:self.scales]]

    def keypoints(self, x_dim: int, y_dim: int) -> int:
        return sum(self.keypoints_per_scale(x_dim, y_dim))

    def _extract(self, batch: ImageBatch) -> ItemBatch:
        if batch.channels != 1:
            raise KeystoneError(-1, "SIFTExtractor: the images must have one channel (apply GrayScaler first)")
        nkp = self.keypoints(batch.x_dim, batch.y_dim)
        h = C.c_int64(0)
        check(batch.ctx.handle, lib().ks_sift_extract(batch.ctx.handle, batch.matrix.handle, batch.x_dim, batch.y_dim, self.step, self.bin,
                                                      self.scales, self.scale_step, C.byref(h)))
        return ItemBatch(_new_matrix(batch.ctx, h.value), np.arange(batch.rows + 1, dtype=np.int64) * nkp)

    def apply(self, data):
        batches, order = _image_batches(self, data)
        if order is None:
            return self._extract(batches[0])
        if order == "single":
            return self._extract(batches[0]).to_list(np.float32)[0]
        if len(batches) == 1 and isinstance(data, (list, tuple)) and not isinstance(data[0], ImageBatch):
            return self._extract(batches[0])
        # several batches: one extraction each, the items put back in input order on the host
        n = sum(len(idx) for idx in order)
        items: List[Optional[np.ndarray]] = [None] * n
        for b, idx in zip(batches, order):
            got = self._extract(b).to_list(np.float32)
            if len(got) != len(idx):
                raise ValueError("SIFTExtractor: an ImageBatch inside a list must hold exactly one image")
            for i, m in zip(idx, got):
                items[i] = m
        return ItemBatch.from_items(batches[0].ctx, items)


# ---------------------------------------------------------------------------------------------------------------- HOG and DAISY
# K/nodes/images/{HogExtractor,DaisyExtractor}.scala.  DESIGN.md section 19.
def _items_in_input_order(node, data, extract, single):
    """extract(ImageBatch) -> ItemBatch over the inputs _image_batches accepts; one image gives single(that ItemBatch), and a list
    that needed several batches is put back in input order on the host."""
    batches, order = _image_batches(node, data)
    if order is None:
        return extract(batches[0])
    if order == "single":
        return single(extract(batches[0]))
    if len(batches) == 1 and isinstance(data, (list, tuple)) and not isinstance(data[0], ImageBatch):
        return extract(batches[0])
    rows: List[Optional[np.ndarray]] = [None] * sum(len(idx) for idx in order)
    for b, idx in zip(batches, order):
        got = extract(b)
        if got.n_items != len(idx):
            raise ValueError(f"{type(node).__name__}: an ImageBatch inside a list must hold exactly one image")
        host = got.to_numpy(np.float32)
        for k, i in enumerate(idx):
            rows[i] = host[got.offsets[k]:got.offsets[k + 1]]
    return ItemBatch(batches[0].ctx.matrix(np.concatenate(rows, 0)), np.cumsum([0] + [r.shape[0] for r in rows]))


def _item_batch(batch: ImageBatch, handle: int) -> ItemBatch:
    m = _new_matrix(batch.ctx, handle)
    per = m.rows // batch.rows if batch.rows else 0
    return ItemBatch(m, np.arange(batch.rows + 1, dtype=np.int64) * per)


class HogExtractor(Transformer):
    """``new HogExtractor(binSize)`` (K/nodes/images/HogExtractor.scala, voc-release5's features.cc): per interior cell of
    round(xDim / bin) x round(yDim / bin) cells, 18 contrast-sensitive, 9 contrast-insensitive and 4 texture values and a zero.
    Input: three-channel BGR images, usually PixelScaler's output (its x / 255.0 is then taken in fp64 with the gradients, as the
    reference never rounds it) -- an ``ImageBatch``, an (n, x, y, 3) array, one (x, y, 3) image (returns the reference's (cells x 32)
    matrix) or a list of images, grouped by shape, input order kept.  Output: an ``ItemBatch`` with one item per image and one cell
    per row, row y + x (nY - 2)."""

    numFeatures = 32

    def __init__(self, binSize: int, ctx: Optional[Context] = None):
        self.bin, self.ctx = int(binSize), ctx

    def cells(self, x_dim: int, y_dim: int) -> int:
        """Feature rows per image: (nX - 2)(nY - 2), with nX = round(x_dim / bin) as Scala rounds (floor(v + 0.5))."""
        nx, ny = (int(np.floor(d / self.bin + 0.5)) for d in (x_dim, y_dim))
        return max(nx - 2, 0) * max(ny - 2, 0)

    def _extract(self, batch: ImageBatch) -> ItemBatch:
        scaled = isinstance(batch, _PixelScaledImages) and batch._matrix is None
        src = batch.source if scaled else batch
        h = C.c_int64(0)
        check(batch.ctx.handle, lib().ks_hog_extract(batch.ctx.handle, src.matrix.handle, batch.x_dim, batch.y_dim, batch.channels,
                                                     1 if scaled else 0, self.bin, C.byref(h)))
        return _item_batch(batch, h.value)

    def apply(self, data):
        return _items_in_input_order(self, data, self._extract, lambda items: items.to_numpy(np.float32))


class DaisyExtractor(Transformer):
    """``new DaisyExtractor(daisyT, daisyQ, daisyR, daisyH, pixelBorder, stride, patchSize)`` (K/nodes/images/DaisyExtractor.scala):
    per keypoint (x = pixelBorder .. xDim - pixelBorder - 1 by stride outer, y likewise inner) the centre histogram and daisyT x daisyQ
    ring histograms of daisyH rectified, Gaussian-blurred orientation maps, each L2-normalised in fp64 (``daisyFeatureSize`` =
    daisyH (daisyT daisyQ + 1) values).  ``patchSize`` is unused, as in the reference.  Input: one-channel images (GrayScaler's
    output), accepted as by ``SIFTExtractor``; one image returns its (daisyFeatureSize x nKP) matrix, as the reference.  Output: an
    ``ItemBatch`` with one item per image, one keypoint per row."""

    def __init__(self, daisyT: int = 8, daisyQ: int = 3, daisyR: int = 7, daisyH: int = 8, pixelBorder: int = 16, stride: int = 4,
                 patchSize: int = 24, ctx: Optional[Context] = None):
        self.daisyT, self.daisyQ, self.daisyR, self.daisyH = int(daisyT), int(daisyQ), int(daisyR), int(daisyH)
        self.pixelBorder, self.stride, self.patchSize, self.ctx = int(pixelBorder), int(stride), int(patchSize), ctx
        self.daisyFeatureSize = self.daisyH * (self.daisyT * self.daisyQ + 1)

    def keypoints(self, x_dim: int, y_dim: int) -> int:
        return len(range(self.pixelBorder, x_dim - self.pixelBorder, self.stride)) * \
            len(range(self.pixelBorder, y_dim - self.pixelBorder, self.stride))

    def _extract(self, batch: ImageBatch) -> ItemBatch:
        h = C.c_int64(0)
        check(batch.ctx.handle, lib().ks_daisy_extract(batch.ctx.handle, batch.matrix.handle, batch.x_dim, batch.y_dim, self.daisyT,
                                                       self.daisyQ, self.daisyR, self.daisyH, self.pixelBorder, self.stride, C.byref(h)))
        return _item_batch(batch, h.value)

    def apply(self, data):
        return _items_in_input_order(self, data, self._extract, lambda items: items.to_list(np.float32)[0])


# ------------------------------------------------------------------------------------------------- image views and augmentation
# Windower, Cropper, RandomPatcher, CenterCornerPatcher and RandomImageTransformer (K/nodes/images/*.scala) as tables of views of a
# source ImageBatch, and Sampler / MatrixUtils.sampleRows (K/nodes/stats/Sampling.scala, K/utils/MatrixUtils.scala).  Only index
# bookkeeping runs on the host; every pixel is moved by ks_image_views or by the Convolver reading the views.  DESIGN.md section 21.
class JavaRandom:
    """``java.util.Random(seed)``: the 48-bit linear congruential generator, ``nextInt``, ``nextInt(bound)`` and ``nextDouble``
    exactly as the JDK defines them, so that seeded draws match the reference's."""

    _MULT, _ADD, _MASK = 0x5DEECE66D, 0xB, (1 << 48) - 1

    def __init__(self, seed: int):
        self._seed = (int(seed) ^ self._MULT) & self._MASK

    def _next(self, bits: int) -> int:
        self._seed = (self._seed * self._MULT + self._ADD) & self._MASK
        r = self._seed >> (48 - bits)
        return r - (1 << 32) if r >= (1 << 31) else r          # (int) of the top bits

    def nextInt(self, bound: Optional[int] = None) -> int:
        if bound is None:
            return self._next(32)
        bound = int(bound)
        if bound <= 0:
            raise ValueError("bound must be positive")
        r = self._next(31)
        m = bound - 1
        if bound & m == 0:                                     # a power of two
            return (bound * r) >> 31
        u = r
        r = u % bound
        while u - r + m >= (1 << 31):                          # u - r + m overflows int: reject and draw again
            u = self._next(31)
            r = u % bound
        return r

    def nextDouble(self) -> float:
        return ((self._next(26) << 27) + self._next(27)) * (1.0 / (1 << 53))


class _FlipHorizontal:
    """``ImageUtils.flipHorizontal``: reverses every image along y (ImageUtils.scala:399-420)."""

    def __repr__(self) -> str:
        return "flip_horizontal"


flip_horizontal = _FlipHorizontal()


class ImageViews(ImageBatch):
    """Views of a source ``ImageBatch``, all ``x_dim`` x ``y_dim``: ``views`` is an (n x 4) int32 table (src_row, x0, y0, flip), view v
    being ``ImageUtils.crop(src, x0, y0, x0 + x_dim, y0 + y_dim)``, reversed along y when flip is 1.  Lazy: ``matrix`` (and
    ``ImageVectorizer`` / ``to_numpy``) gathers the views on the device; a ``Convolver`` reads them without materialising them."""

    def __init__(self, source: ImageBatch, views, x_dim: int, y_dim: int):
        views = np.ascontiguousarray(views, dtype=np.int32).reshape(-1, 4)
        self.ctx, self.source, self.views = source.ctx, source, views
        self.x_dim, self.y_dim, self.channels = int(x_dim), int(y_dim), source.channels
        self._matrix: Optional[DeviceMatrix] = None

    @property
    def rows(self) -> int:
        return int(self.views.shape[0])

    @property
    def matrix(self) -> DeviceMatrix:
        if self._matrix is None:
            s = self.source
            h = C.c_int64(0)
            check(self.ctx.handle, lib().ks_image_views(self.ctx.handle, s.matrix.handle, s.x_dim, s.y_dim, s.channels,
                                                        self.views.ctypes.data_as(C.c_void_p), self.rows, self.x_dim, self.y_dim,
                                                        C.byref(h)))
            self._matrix = DeviceMatrix(self.ctx, h.value, self.rows, self.x_dim * self.y_dim * self.channels)
        return self._matrix

    def materialize(self) -> DeviceMatrix:
        return self.matrix

    def to_numpy(self, dtype=np.float64) -> np.ndarray:
        return self.matrix.to_numpy(dtype)

    def take(self, rows) -> "ImageViews":
        """The views at these positions of the table, in that order (nothing is gathered)."""
        return ImageViews(self.source, self.views[np.asarray(rows, dtype=np.int64)], self.x_dim, self.y_dim)


def _view_base(node, data):
    """(source batch, its (n x 4) views, x_dim, y_dim): an ImageViews as it is, any other image batch as one whole view per image."""
    if isinstance(data, ImageViews):
        return data.source, data.views, data.x_dim, data.y_dim
    if not isinstance(data, ImageBatch):
        data = _image_batches(node, data)[0][0]
    n = data.rows
    base = np.zeros((n, 4), dtype=np.int32)
    base[:, 0] = np.arange(n)
    return data, base, data.x_dim, data.y_dim


def _crop_views(node, data, local: np.ndarray, out_x: int, out_y: int) -> ImageViews:
    """local: (m x 4) (image, x0, y0, flip) relative to the input images (image = row of the input batch); composed with the
    input's own views so that the result is a table of views of the source batch."""
    src, base, x_dim, y_dim = _view_base(node, data)
    local = np.asarray(local, dtype=np.int64).reshape(-1, 4)
    if local.size and ((local[:, 1] < 0).any() or (local[:, 1] + out_x > x_dim).any() or (local[:, 2] < 0).any()
                       or (local[:, 2] + out_y > y_dim).any() or out_x < 1 or out_y < 1):
        raise KeystoneError(-1, "invalid crop: the view leaves the image")
    b = base[local[:, 0]].astype(np.int64)
    flipped = b[:, 3] == 1
    out = np.empty_like(local)
    out[:, 0] = b[:, 0]
    out[:, 1] = b[:, 1] + local[:, 1]
    # a crop of a flipped view is the mirrored range of the source, still flipped
    out[:, 2] = np.where(flipped, b[:, 2] + y_dim - local[:, 2] - out_y, b[:, 2] + local[:, 2])
    out[:, 3] = b[:, 3] ^ local[:, 3]
    return ImageViews(src, out, out_x, out_y)


class Windower(Transformer):
    """``new Windower(stride, windowSize)`` (K/nodes/images/Windower.scala): every windowSize x windowSize window at x, y = 0, stride,
    ... <= dim - windowSize, x outer and y inner, per image in order.  Returns ``ImageViews``."""

    def __init__(self, stride: int, windowSize: int, ctx: Optional[Context] = None):
        self.stride, self.window, self.ctx = int(stride), int(windowSize), ctx
        if self.stride < 1 or self.window < 1:
            raise ValueError("stride and windowSize must be >= 1")

    def views(self, n_images: int, x_dim: int, y_dim: int) -> np.ndarray:
        xs = np.arange(0, x_dim - self.window + 1, self.stride)
        ys = np.arange(0, y_dim - self.window + 1, self.stride)
        per = np.stack([np.repeat(xs, ys.size), np.tile(ys, xs.size)], 1)
        out = np.zeros((n_images * per.shape[0], 4), dtype=np.int64)
        out[:, 0] = np.repeat(np.arange(n_images), per.shape[0])
        out[:, 1:3] = np.tile(per, (n_images, 1))
        return out

    def apply(self, data) -> ImageViews:
        _, base, x_dim, y_dim = _view_base(self, data)
        return _crop_views(self, data, self.views(base.shape[0], x_dim, y_dim), self.window, self.window)


class Cropper(Transformer):
    """``Cropper(startX, startY, endX, endY)`` (K/nodes/images/Cropper.scala): ``ImageUtils.crop`` of every image."""

    def __init__(self, startX: int, startY: int, endX: int, endY: int, ctx: Optional[Context] = None):
        self.sx, self.sy, self.ex, self.ey, self.ctx = int(startX), int(startY), int(endX), int(endY), ctx

    def apply(self, data) -> ImageViews:
        _, base, _, _ = _view_base(self, data)
        n = base.shape[0]
        local = np.stack([np.arange(n), np.full(n, self.sx), np.full(n, self.sy), np.zeros(n, dtype=np.int64)], 1)
        return _crop_views(self, data, local, self.ex - self.sx, self.ey - self.sy)


class RandomPatcher(Transformer):
    """``RandomPatcher(numPatches, patchSizeX, patchSizeY, seed)`` (K/nodes/images/RandomPatcher.scala): per image, numPatches crops
    with ``startX = rnd.nextInt(xDim - patchSizeX + 1)`` and then ``startY = rnd.nextInt(yDim - patchSizeY + 1)``, ``rnd`` a
    ``java.util.Random(seed)``.  Spark hands every partition a fresh copy of the node, so the stream restarts from the seed on each
    partition; here it restarts on every call, a call being one rank's shard.  Returns ``ImageViews``."""

    def __init__(self, numPatches: int, patchSizeX: int, patchSizeY: int, seed: int = 12334, ctx: Optional[Context] = None):
        self.n, self.px, self.py, self.seed, self.ctx = int(numPatches), int(patchSizeX), int(patchSizeY), int(seed), ctx

    def views(self, n_images: int, x_dim: int, y_dim: int) -> np.ndarray:
        if self.px > x_dim or self.py > y_dim or self.px < 1 or self.py < 1:
            raise KeystoneError(-1, "RandomPatcher: the patch must fit in the image")
        rnd = JavaRandom(self.seed)
        out = np.zeros((n_images * self.n, 4), dtype=np.int64)
        for v in range(n_images * self.n):
            out[v, 0] = v // self.n
            out[v, 1] = rnd.nextInt(x_dim - self.px + 1)
            out[v, 2] = rnd.nextInt(y_dim - self.py + 1)
        return out

    def apply(self, data) -> ImageViews:
        _, base, x_dim, y_dim = _view_base(self, data)
        return _crop_views(self, data, self.views(base.shape[0], x_dim, y_dim), self.px, self.py)


class CenterCornerPatcher(Transformer):
    """``CenterCornerPatcher(patchSizeX, patchSizeY, horizontalFlips)`` (K/nodes/images/CenterCornerPatcher.scala): per image the
    crops at the four corners and the centre, in the reference's order, each followed by its flip when ``horizontalFlips``."""

    def __init__(self, patchSizeX: int, patchSizeY: int, horizontalFlips: bool, ctx: Optional[Context] = None):
        self.px, self.py, self.flips, self.ctx = int(patchSizeX), int(patchSizeY), bool(horizontalFlips), ctx

    def views(self, n_images: int, x_dim: int, y_dim: int) -> np.ndarray:
        bx, by = x_dim - self.px, y_dim - self.py
        starts = [(0, 0), (bx, 0), (0, by), (bx, by), (bx // 2, by // 2)]
        per = [(x, y, f) for x, y in starts for f in ((0, 1) if self.flips else (0,))]
        out = np.zeros((n_images * len(per), 4), dtype=np.int64)
        out[:, 0] = np.repeat(np.arange(n_images), len(per))
        out[:, 1:] = np.tile(np.asarray(per, dtype=np.int64), (n_images, 1))
        return out

    def apply(self, data) -> ImageViews:
        _, base, x_dim, y_dim = _view_base(self, data)
        return _crop_views(self, data, self.views(base.shape[0], x_dim, y_dim), self.px, self.py)


class RandomImageTransformer(Transformer):
    """``RandomImageTransformer(chance, transform, seed)`` (K/nodes/images/RandomImageTransformer.scala): per image in order, the
    transform applies when ``rnd.nextDouble() < chance``, ``rnd`` a ``java.util.Random(seed)`` restarted on every call (one rank's
    shard, as RandomPatcher).  The transform must be ``flip_horizontal``, which toggles the flip of a view; there is no host path
    for any other function.  Returns ``ImageViews``."""

    def __init__(self, chance: float, transform, seed: int = 12334, ctx: Optional[Context] = None):
        if transform is not flip_horizontal:
            raise KeystoneError(-1, "RandomImageTransformer: only flip_horizontal runs on the device")
        self.chance, self.transform, self.seed, self.ctx = float(chance), transform, int(seed), ctx

    def flips(self, n: int) -> np.ndarray:
        rnd = JavaRandom(self.seed)
        return np.array([1 if rnd.nextDouble() < self.chance else 0 for _ in range(n)], dtype=np.int32)

    def apply(self, data) -> ImageViews:
        src, base, x_dim, y_dim = _view_base(self, data)
        views = base.copy()
        views[:, 3] ^= self.flips(views.shape[0])
        return ImageViews(src, views, x_dim, y_dim)


def _sample_indices(n: int, size: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).choice(n, min(int(size), n), replace=False).astype(np.int64)


class Sampler(Transformer):
    """``new Sampler(size, seed)`` (K/nodes/stats/Sampling.scala): ``takeSample(false, size, seed)``.  Spark's draw depends on the
    partitioning and is not reproduced: the rows are ``numpy.random.default_rng(seed).choice(n, min(size, n), replace=False)``.  On
    ``ImageViews`` the view table is subset before anything is gathered; on a device matrix the rows are gathered on the device."""

    def __init__(self, size: int, seed: int = 42, ctx: Optional[Context] = None):
        self.size, self.seed, self.ctx = int(size), int(seed), ctx

    def apply(self, data):
        if isinstance(data, ImageViews):
            return data.take(_sample_indices(data.rows, self.size, self.seed))
        x = _device_matrix(self.ctx, data)
        return _gather_rows(x, _sample_indices(x.rows, self.size, self.seed))


def sample_rows(data, num_samples: int, seed: int = 42, ctx: Optional[Context] = None) -> DeviceMatrix:
    """``MatrixUtils.sampleRows`` (K/utils/MatrixUtils.scala:116-119): ``num_samples`` distinct rows, drawn as by ``Sampler``
    (the reference's unseeded ``Random.shuffle`` is not reproduced) and kept in ascending order as the reference sorts them."""
    x = _device_matrix(ctx, data)
    return _gather_rows(x, np.sort(_sample_indices(x.rows, num_samples, seed)))


def _gather_rows(x: DeviceMatrix, rows: np.ndarray) -> DeviceMatrix:
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    h = C.c_int64(0)
    check(x.ctx.handle, lib().ks_matrix_gather_rows(x.ctx.handle, x.handle, rows.ctypes.data_as(C.c_void_p), rows.size, C.byref(h)))
    return DeviceMatrix(x.ctx, h.value, rows.size, x.cols)


# ------------------------------------------------------------------------------------------ the text front end (DESIGN.md section 23)
def _as_text(ctx: Optional[Context], data) -> TextBatch:
    if isinstance(data, TextBatch):
        return data
    if isinstance(data, Dataset):
        raise KeystoneError(-1, f"a text node needs a TextBatch, not {type(data).__name__}")
    if ctx is None:
        raise KeystoneError(-1, "host documents need a Context (pass ctx= to the node)")
    return ctx.text(list(data))


def _as_terms(ctx: Optional[Context], data):
    """(token batch, min order, max order) of a batch of terms: a ``TokenBatch`` (its tokens as terms, orders 0, 0), an ``NGramBatch``,
    or host lists of ``str`` tokens.  Host lists of n-gram tuples are rejected: n-grams reach the device as an ``NGramBatch``."""
    if isinstance(data, NGramBatch):
        return data.tokens, data.min_order, data.max_order
    if isinstance(data, TokenBatch):
        return data, 0, 0
    if isinstance(data, Dataset):
        raise KeystoneError(-1, f"a term node needs a TokenBatch or an NGramBatch, not {type(data).__name__}")
    if ctx is None:
        raise KeystoneError(-1, "host token lists need a Context (pass ctx= to the node)")
    docs = [list(d) for d in data]
    if any(isinstance(t, tuple) for d in docs for t in d):
        # the device emits n-grams from tokens; arbitrary host tuples have no token batch and orders to be emitted from
        raise KeystoneError(-1, "host lists of n-gram tuples are not accepted: pass the tokens through NGramsFeaturizer, which gives "
                                "an NGramBatch")
    return ctx.tokens(docs), 0, 0


def _as_tf(ctx: Optional[Context], data) -> TermFrequencyBatch:
    if isinstance(data, TermFrequencyBatch):
        return data
    if isinstance(data, Dataset):
        raise KeystoneError(-1, f"this node needs a TermFrequencyBatch, not {type(data).__name__}")
    if ctx is None:
        raise KeystoneError(-1, "host term-frequency lists need a Context (pass ctx= to the node)")
    return ctx.term_frequencies([list(d) for d in data])


def _check_orders(orders) -> tuple:
    """NGramsFeaturizer's requirements (ngrams.scala): orders >= 1 and consecutive, in increasing order."""
    o = [int(x) for x in orders]
    if not o:
        raise ValueError("orders must not be empty")
    if min(o) < 1:
        raise ValueError(f"minimum order is not >= 1, found {min(o)}")
    for a, b in zip(o, o[1:]):
        if a != b - 1:
            raise ValueError(f"orders are not consecutive; contains {a} and {b}")
    return o[0], o[-1]


def _sparse_result(ctx: Context, handle: int) -> SparseMatrix:
    rows, cols, nnz = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    check(ctx.handle, lib().ks_sparse_shape(ctx.handle, handle, C.byref(rows), C.byref(cols), C.byref(nnz)))
    return SparseMatrix(ctx, handle, rows.value, cols.value, nnz.value)


def _transform_text(ctx: Optional[Context], data, flags: int) -> TextBatch:
    t = _as_text(ctx, data)
    h = C.c_int64(0)
    check(t.ctx.handle, lib().ks_text_transform(t.ctx.handle, t.handle, flags, C.byref(h)))
    return TextBatch(t.ctx, h.value, t.n_docs)


class Trim(Transformer):
    """``Trim`` (K/nodes/nlp/StringUtils.scala): Java's ``String.trim``, which strips leading and trailing code points <= U+0020."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    def apply(self, data) -> TextBatch:
        return _transform_text(self.ctx, data, _capi.KS_TEXT_TRIM)


class LowerCase(Transformer):
    """``LowerCase(locale)`` (K/nodes/nlp/StringUtils.scala) in the root locale: every code point by its one-to-one Unicode lowercase
    mapping, and U+0130 to "i" U+0307 as Java does.  Java's final-sigma rule is not applied (a final capital sigma becomes U+03C3).
    The Turkish, Azeri and Lithuanian locales, whose rules differ, are rejected."""

    def __init__(self, locale: Optional[str] = None, ctx: Optional[Context] = None):
        if locale is not None and str(locale).replace("-", "_").split("_")[0].lower() in ("tr", "az", "lt"):
            raise ValueError(f"LowerCase: the {locale} locale has its own lowercase rules, which are not implemented")
        self.locale, self.ctx = locale, ctx

    def apply(self, data) -> TextBatch:
        return _transform_text(self.ctx, data, _capi.KS_TEXT_LOWER)


class Tokenizer(Transformer):
    """``Tokenizer(sep)`` (K/nodes/nlp/StringUtils.scala) with the default pattern ``[\\p{Punct}\\s]+`` only: Java's
    ``String.split`` on runs of ASCII punctuation and whitespace.  A leading separator gives a leading "", trailing empty strings
    are dropped, "" gives [""] and a document of separators only gives []."""

    DEFAULT_SEP = "[\\p{Punct}\\s]+"

    def __init__(self, sep: str = DEFAULT_SEP, ctx: Optional[Context] = None):
        if sep != self.DEFAULT_SEP:
            raise ValueError(f"Tokenizer: only the default separator {self.DEFAULT_SEP!r} is implemented, not {sep!r}")
        self.sep, self.ctx = sep, ctx

    def apply(self, data) -> TokenBatch:
        t = _as_text(self.ctx, data)
        h = C.c_int64(0)
        check(t.ctx.handle, lib().ks_text_tokenize(t.ctx.handle, t.handle, C.byref(h)))
        return TokenBatch(t.ctx, h.value, t.n_docs)


class NGramsFeaturizer(Transformer):
    """``NGramsFeaturizer(orders)`` (K/nodes/nlp/ngrams.scala): the n-grams of every document as tuples, for each position i and
    then each order.  The result is an ``NGramBatch``, emitted on the device by the node that consumes it; ``TermFrequency`` takes
    orders up to 4, the hashing nodes any order."""

    def __init__(self, orders, ctx: Optional[Context] = None):
        self.min_order, self.max_order = _check_orders(orders)
        self.orders, self.ctx = list(range(self.min_order, self.max_order + 1)), ctx

    def apply(self, data) -> NGramBatch:
        tokens, mn, _ = _as_terms(self.ctx, data)
        if mn != 0:
            raise KeystoneError(-1, "NGramsFeaturizer takes tokens, not n-grams")
        return NGramBatch(tokens, self.min_order, self.max_order)


def _identity(x):
    return x


class TermFrequency(Transformer):
    """``TermFrequency(fun)`` (K/nodes/stats/TermFrequency.scala): per document its distinct terms, in order of first occurrence,
    each with ``fun(count)``.  The device counts; ``fun`` is evaluated on the host once for every count 1 .. the largest count in the
    batch, and a result that is not finite is rejected.  Input: a ``TokenBatch``, an ``NGramBatch`` or host lists of ``str`` tokens
    (host lists of n-gram tuples are rejected; use ``NGramsFeaturizer`` on the tokens)."""

    def __init__(self, fun=_identity, ctx: Optional[Context] = None):
        self.fun, self.ctx = fun, ctx

    def apply(self, data) -> TermFrequencyBatch:
        tokens, mn, mx = _as_terms(self.ctx, data)
        ctx = tokens.ctx
        h, mc = C.c_int64(0), C.c_int64(0)
        check(ctx.handle, lib().ks_term_frequency(ctx.handle, tokens.handle, mn, mx, C.byref(h), C.byref(mc)))
        tf = TermFrequencyBatch(ctx, h.value, tokens.n_docs, tokens, mc.value)
        if self.fun is not _identity and mc.value > 0:
            table = np.array([float(self.fun(float(c))) for c in range(1, mc.value + 1)], dtype=np.float64)
            bad = np.flatnonzero(~np.isfinite(table))
            if bad.size:
                raise KeystoneError(-1, f"TermFrequency: fun({int(bad[0]) + 1}) = {table[bad[0]]} is not finite")
            check(ctx.handle, lib().ks_tf_set_weights(ctx.handle, tf.handle, table.ctypes.data_as(C.c_void_p), table.shape[0]))
        return tf


class SparseFeatureVectorizer(Transformer):
    """``SparseFeatureVectorizer(featureSpace)`` (K/nodes/util/SparseFeatureVectorizer.scala): ``apply`` maps every document's
    ``(term, value)`` pairs to a ``SparseMatrix`` row with ``len(feature_space)`` columns, fp64 values, columns ascending; terms
    outside the space are dropped, and a term repeated within one document of a host list gives one entry, the sum of its values.  Terms match by their bytes.  ``SparseFeatureVectorizer(feature_space, ctx=ctx)`` uploads a host
    ``{term: column}`` dict whose columns are 0 .. n-1; ``feature_space`` reads the fitted space back as such a dict."""

    def __init__(self, feature_space, ctx: Optional[Context] = None, _handle: int = 0):
        if _handle:
            self.ctx, self.handle = ctx, _handle
            n = C.c_int64(0)
            check(ctx.handle, lib().ks_text_array_size(ctx.handle, _handle, _capi.KS_TEXT_TERM_ORDER, C.byref(n)))
            self.num_features = n.value
            return
        if ctx is None:
            raise KeystoneError(-1, "SparseFeatureVectorizer from a host feature space needs a Context (pass ctx=)")
        items = sorted(dict(feature_space).items(), key=lambda kv: kv[1])
        if [v for _, v in items] != list(range(len(items))):
            raise ValueError("the feature space's columns must be 0 .. len(feature_space) - 1")
        tokens, first, order = _flatten_terms([k for k, _ in items])
        tk = ctx.tokens([tokens])
        h = C.c_int64(0)
        check(ctx.handle, lib().ks_sparse_features_from_host(ctx.handle, tk.handle, first.ctypes.data_as(C.c_void_p),
                                                              order.ctypes.data_as(C.c_void_p), len(items), C.byref(h)))
        self.ctx, self.handle, self.num_features = ctx, h.value, len(items)

    @property
    def feature_space(self) -> dict:
        return {t: i for i, t in enumerate(_host_terms(self.ctx, self.handle))}

    def apply(self, data) -> SparseMatrix:
        tf = _as_tf(self.ctx, data)
        h = C.c_int64(0)
        check(self.ctx.handle, lib().ks_sparse_features_apply(self.ctx.handle, self.handle, tf.handle, C.byref(h)))
        return _sparse_result(self.ctx, h.value)

    def __del__(self):
        try:
            if self.handle and self.ctx.handle:
                lib().ks_text_destroy(self.ctx.handle, self.handle)
        except Exception:
            pass


def _fit_space(ctx: Optional[Context], data, num_features: int) -> SparseFeatureVectorizer:
    tf = _as_tf(ctx, data)
    if tf.ctx.world_size > 1:
        raise KeystoneError(-1, "CommonSparseFeatures / AllSparseFeatures fit on one rank only: an exact top-K over ranks is not implemented")
    h = C.c_int64(0)
    check(tf.ctx.handle, lib().ks_sparse_features_fit(tf.ctx.handle, tf.handle, num_features, C.byref(h)))
    return SparseFeatureVectorizer(None, tf.ctx, _handle=h.value)


class CommonSparseFeatures(Estimator):
    """``CommonSparseFeatures(numFeatures)`` (K/nodes/util/CommonSparseFeatures.scala): ``fit`` keeps the ``num_features`` terms
    held by the most entries (document frequency), ties by earliest appearance in the flattened batch, and returns a
    ``SparseFeatureVectorizer``.  One rank only."""

    def __init__(self, num_features: int, ctx: Optional[Context] = None):
        if int(num_features) < 1:
            raise ValueError("num_features must be >= 1")
        self.num_features, self.ctx = int(num_features), ctx

    def fit(self, data) -> SparseFeatureVectorizer:
        return _fit_space(self.ctx, data, self.num_features)


class AllSparseFeatures(Estimator):
    """``AllSparseFeatures()`` (K/nodes/util/AllSparseFeatures.scala): every term, in the order of ``CommonSparseFeatures`` without a
    cut.  One rank only."""

    def __init__(self, ctx: Optional[Context] = None):
        self.ctx = ctx

    def fit(self, data) -> SparseFeatureVectorizer:
        return _fit_space(self.ctx, data, -1)


def _hashing_tf(ctx: Optional[Context], data, num_features: int, orders=None) -> SparseMatrix:
    tokens, mn, mx = _as_terms(ctx, data)
    if orders is not None:
        if mn != 0:
            raise KeystoneError(-1, "NGramsHashingTF takes tokens, not n-grams")
        mn, mx = orders
    h = C.c_int64(0)
    check(tokens.ctx.handle, lib().ks_hashing_tf(tokens.ctx.handle, tokens.handle, mn, mx, num_features, C.byref(h)))
    return _sparse_result(tokens.ctx, h.value)


class HashingTF(Transformer):
    """``HashingTF(numFeatures)`` (K/nodes/nlp/HashingTF.scala): term counts at column ``nonNegativeMod(term.##, numFeatures)``:
    ``String.hashCode`` for the tokens of a ``TokenBatch`` (or host lists of ``str``), ``MurmurHash3.seqHash`` for the tuples of an
    ``NGramBatch``.  Host lists of n-gram tuples are rejected; use ``NGramsFeaturizer`` on the tokens."""

    def __init__(self, num_features: int, ctx: Optional[Context] = None):
        if not 1 <= int(num_features) < 2 ** 31:
            raise ValueError("num_features must lie in [1, 2^31 - 1]")
        self.num_features, self.ctx = int(num_features), ctx

    def apply(self, data) -> SparseMatrix:
        return _hashing_tf(self.ctx, data, self.num_features)


class NGramsHashingTF(Transformer):
    """``NGramsHashingTF(orders, numFeatures)`` (K/nodes/nlp/NGramsHashingTF.scala): the same counts as ``NGramsFeaturizer(orders)
    andThen HashingTF(numFeatures)`` without forming the n-grams; any order."""

    def __init__(self, orders, num_features: int, ctx: Optional[Context] = None):
        self.min_order, self.max_order = _check_orders(orders)
        if not 1 <= int(num_features) < 2 ** 31:
            raise ValueError("num_features must lie in [1, 2^31 - 1]")
        self.num_features, self.ctx = int(num_features), ctx

    def apply(self, data) -> SparseMatrix:
        return _hashing_tf(self.ctx, data, self.num_features, (self.min_order, self.max_order))
