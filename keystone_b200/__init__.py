"""keystone_b200 -- H100-native block least-squares engine behind the KeystoneML node API.

The package is a thin host layer over ``lib/libkeystone_b200.so`` (C ABI in ``include/keystone_b200.h``);
all numerics run in hand-written sm_90a kernels.  There is no CPU fallback.
"""
from ._capi import KeystoneError, LIB_PATH, declared_symbols  # noqa: F401
from .context import Context, DeviceMatrix, LazyFeatures, shard_range  # noqa: F401
from .workflow import Estimator, LabelEstimator, Pipeline, Transformer  # noqa: F401
from .nodes import (  # noqa: F401
    ApproximatePCAEstimator,
    BatchPCATransformer,
    ColumnPCAEstimator,
    DistributedColumnPCAEstimator,
    DistributedPCAEstimator,
    LocalColumnPCAEstimator,
    PCAEstimator,
    PCATransformer,
    ZCAWhitener,
    ZCAWhitenerEstimator,
    BatchSignedHellingerMapper,
    FisherVector,
    FloatToDouble,
    GaussianMixtureModel,
    ImageBatch,
    ItemBatch,
    LCSExtractor,
    MatrixVectorizer,
    NormalizeRows,
    SignedHellingerMapper,
    BlockLeastSquaresEstimator,
    BlockLinearMapper,
    BlockWeightedLeastSquaresEstimator,
    ClassLabelIndicatorsFromIntLabels,
    Convolver,
    CosineRandomFeatures,
    DenseLBFGSwithL2,
    GaussianKernelGenerator,
    GaussianKernelTransformer,
    ImageVectorizer,
    KernelBlockLinearMapper,
    KernelMatrix,
    KernelRidgeRegression,
    Pooler,
    SymmetricRectifier,
    cifar_bytes_to_matrix,
    images_to_matrix,
    LeastSquaresDenseGradient,
    LeastSquaresEstimator,
    LinearMapEstimator,
    LinearMapper,
    LinearRectifier,
    MaxClassifier,
    PaddedFFT,
    RandomSignNode,
    VectorCombiner,
    VectorSplitter,
)
from .loaders import (  # noqa: F401
    CifarLoader,
    CsvDataLoader,
    LabeledData,
    MnistCsvLoader,
    TimitFeaturesDataLoader,
    TimitLabelsLoader,
)
from .evaluation import (  # noqa: F401
    BinaryClassificationMetrics,
    MulticlassClassifierEvaluator,
    MulticlassMetrics,
)
