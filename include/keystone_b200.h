/* keystone_b200 -- C ABI of the H100-native (sm_90a) block least-squares engine.
 *
 * Drop-in boundary for the KeystoneML (amplab/keystone) node bodies on the block-LS hot path.
 * Every entry point names the reference interface it replaces (paths relative to
 * /root/reference; K/ = src/main/scala/keystoneml/).  The reference reaches native code
 * through JNI with primitives and primitive arrays only (K/utils/external/VLFeat.scala:18-26,
 * src/main/cpp/VLFeat.cxx:203); this ABI keeps that shape: plain pointers, sizes and opaque
 * 64-bit handles (1:1 with a JVM Long).  INTEGRATION.md shows the JNI / ctypes bindings.
 *
 * Process model: ONE process (context) per GPU.  A row-sharded dataset is represented by every
 * rank holding a matrix handle for ITS rows (the analogue of an RDD partition set); reductions
 * that Spark does with treeReduce (K/nodes/learning/BlockWeightedLeastSquares.scala:212-225,
 * K/utils/MatrixUtils.scala:137-146) are NCCL all-reduces inside the fit calls, so every rank
 * must call the same collective entry points in the same order.
 *
 * Conventions
 *   - every function returns 0 on success, < 0 on error; ks_last_error() gives the message.
 *     Nothing calls exit() or throws across the boundary (the reference's JNI code does
 *     exit(-1), src/main/cpp/EncEval.cxx:43-47).
 *   - host buffers are caller-owned and only borrowed for the duration of the call;
 *     device objects are library-owned and released by the matching *_destroy.
 *   - a context is not thread-safe (same contract as Pipeline / GraphExecutor,
 *     K/workflow/Pipeline.scala:14).
 *   - dense host matrices are row-major with an explicit leading dimension, except where a
 *     parameter says "colmajor": those are Breeze DenseMatrix[Double] layouts (column-major),
 *     so a JVM caller can pass DenseMatrix.data unchanged.
 *   - there is NO CPU fallback: without a CUDA device ks_ctx_create fails.
 */
#ifndef KEYSTONE_B200_H
#define KEYSTONE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define KS_API __attribute__((visibility("default")))
#else
#define KS_API
#endif

#define KS_OK 0
#define KS_ERR_INVALID (-1)
#define KS_ERR_CUDA (-2)
#define KS_ERR_NCCL (-3)
#define KS_ERR_SOLVER (-4)
#define KS_ERR_NO_DEVICE (-5)
#define KS_ERR_HANDLE (-6)
#define KS_ERR_NOT_SPD (-7)

/* precision_mode of the fit entry points.  All modes accumulate in fp32 inside the tensor core, assemble and solve the
 * reduced b x b systems in fp64 (centring correction, Cholesky, triangular solves) and keep the model in fp64. */
#define KS_PRECISION_DEFAULT (-1) /* the context's setting (ks_ctx_set_option "precision"; initial value KS_PRECISION_F16X2) */
#define KS_PRECISION_TF32 0  /* one tf32 MMA per product: operands rounded to tf32 (10-bit mantissa, round-to-nearest) */
#define KS_PRECISION_F16 1   /* fast mode.  Generated (cosine) features: fp16 operands (same 10-bit mantissa as tf32, residual /
                                increments scaled by device-chosen powers of two), fp16 wgmma at twice the tf32 rate;
                                materialised feature matrices fall back to KS_PRECISION_TF32 */
#define KS_PRECISION_F16X2 2 /* parity mode (split operands): every MMA operand v is carried as hi + lo (hi = round(v),
                                lo = round(v - hi): >= 21 significant bits) and every product keeps hi*hi + hi*lo + lo*hi on the
                                same kernels.  Generated features: fp16 pairs (fp16 MMA, ~3x the fast mode's tensor work);
                                materialised feature matrices: tf32 pairs (tf32 MMA).  Measured against the fp64 oracle:
                                see DESIGN.md section 6 */

#define KS_NCCL_ID_BYTES 128

KS_API int32_t ks_version(void);

/* ---- lifecycle --------------------------------------------------------------------------- */
/* Rank 0 creates the NCCL unique id; the host runtime (Spark driver / torch.distributed / MPI)
 * ships the 128 bytes to the other ranks. */
KS_API int32_t ks_nccl_unique_id(uint8_t* out_id /* KS_NCCL_ID_BYTES */);
/* world_size == 1: nccl_id may be NULL and no communicator is created. */
KS_API int32_t ks_ctx_create(int32_t device_id, int32_t rank, int32_t world_size, const uint8_t* nccl_id, int64_t* out_ctx);
KS_API int32_t ks_ctx_destroy(int64_t ctx);
KS_API const char* ks_last_error(int64_t ctx);
KS_API int32_t ks_ctx_synchronize(int64_t ctx);
/* tunables (defaults in brackets): "gram_chunk_rows" [0 = chosen from the local row count], "sample_rows" [16384: rows per rank
 * for the shift estimate of generated features], "precision" [2 = KS_PRECISION_F16X2: what KS_PRECISION_DEFAULT and the entry
 * points without a precision argument use], "proj_f16" [1: fp16 projection operands in fp16 mode], "shard_solve" [1: triangular solves sharded by
 * right-hand-side columns over the ranks], "reserve_sms" [8], "timing" [1], "pipeline" [1: all tensor-core kernels of a fit on
 * one stream, solve / factor chains beside it; 0: the two-stream arrangement of round 1], "host_mirror" [1: fits copy each
 * finished model block into pinned host memory while they run]; "custom_solve" [-1: automatic -- the library's own DMMA
 * multi-right-hand-side triangular solve kernel when a rank solves <= 512 columns (multi-GPU), cusolverDnDpotrs otherwise; 0 / 1 force], "dyn_tiles" [1: the projection kernel draws its tiles from a
 * counter], "lookahead" [0 = automatic: blocks the residual-independent work runs ahead, 1 on one GPU, 2 on several], "solve_lanes" [4: concurrent per-class solves of the weighted solver],
 * "split_chunk_rows" [4096: rows per accumulation chain of the parity mode's Gram launches; the tensor core's accumulation error grows with
 * the chain, DESIGN.md 6]. */
KS_API int32_t ks_ctx_set_option(int64_t ctx, const char* name, int64_t value);

/* ---- row-sharded matrices (this rank's rows) ---------------------------------------------
 * Replace RDD[DenseVector[Double]] + MatrixUtils.rowsToMatrix packing
 * (K/utils/MatrixUtils.scala:48-93).  Stored on device as fp32 row-major, 128 B aligned rows. */
KS_API int32_t ks_matrix_from_host_f64(int64_t ctx, const double* rowmajor, int64_t n_rows, int64_t n_cols, int64_t ld,
                                int64_t* out_m);
KS_API int32_t ks_matrix_from_host_f32(int64_t ctx, const float* rowmajor, int64_t n_rows, int64_t n_cols, int64_t ld,
                                int64_t* out_m);
/* A zero matrix filled by row ranges afterwards: how an executor uploads its RDD partitions one at a time
 * (mapPartitionsWithIndex + MatrixUtils.rowsToMatrix per partition, K/utils/MatrixUtils.scala:48-93). */
KS_API int32_t ks_matrix_create(int64_t ctx, int64_t n_rows, int64_t n_cols, int64_t* out_m);
KS_API int32_t ks_matrix_write_rows_f64(int64_t ctx, int64_t m, int64_t row0, const double* rowmajor, int64_t n_rows, int64_t ld);
KS_API int32_t ks_matrix_write_rows_f32(int64_t ctx, int64_t m, int64_t row0, const float* rowmajor, int64_t n_rows, int64_t ld);
/* iid N(mean, stddev) generated on the device (benchmarks; counter-based, reproducible per (seed,row,col)). */
KS_API int32_t ks_matrix_synthetic_normal(int64_t ctx, int64_t n_rows, int64_t n_cols, uint64_t seed, int64_t global_row_offset,
                                   double mean, double stddev, int64_t* out_m);
/* ClassLabelIndicatorsFromIntLabels (K/nodes/util/ClassLabelIndicators.scala:15-29): +1 / -1 indicators. */
KS_API int32_t ks_labels_from_classes(int64_t ctx, const int32_t* classes, int64_t n_rows, int32_t num_classes, int64_t* out_m);
KS_API int32_t ks_matrix_shape(int64_t ctx, int64_t m, int64_t* n_rows, int64_t* n_cols);
KS_API int32_t ks_matrix_to_host_f64(int64_t ctx, int64_t m, double* rowmajor_out, int64_t ld);
KS_API int32_t ks_matrix_to_host_f32(int64_t ctx, int64_t m, float* rowmajor_out, int64_t ld);
KS_API int32_t ks_matrix_destroy(int64_t ctx, int64_t m);

/* ---- CosineRandomFeatures (K/nodes/stats/CosineRandomFeatures.scala:19-44) ----------------
 * W is (n_out x n_in) COLUMN-major fp64 exactly as Breeze stores it, b has n_out entries. */
KS_API int32_t ks_cosine_rf_create(int64_t ctx, const double* W_colmajor, const double* b, int64_t n_out, int64_t n_in,
                            int64_t* out_rf);
/* apply(RDD) :25-36 -- materialises cos(X W^T + b) as a new (N x n_out) matrix. */
KS_API int32_t ks_cosine_rf_apply(int64_t ctx, int64_t rf, int64_t x_in, int64_t* out_features);
KS_API int32_t ks_cosine_rf_destroy(int64_t ctx, int64_t rf);

/* RandomSignNode(signs) andThen PaddedFFT() [andThen LinearRectifier(maxVal, alpha)] as one dense feature map
 * (K/nodes/stats/RandomSignNode.scala:11-24, PaddedFFT.scala:13-21, LinearRectifier.scala:12-17; the featurizer of
 * K/pipelines/images/mnist/MnistRandomFFT.scala:40-44): out[f] = max(maxVal, sum_n x[n] signs[n] cos(2 pi f n / P) - alpha),
 * f < P / 2, P = nextPositivePowerOfTwo(n_in).  signs may be NULL (all +1); rectify = 0: no rectifier.  The handle is a feature-map
 * handle like CosineRandomFeatures': ks_cosine_rf_apply materialises it, the fits regenerate it block by block, and
 * ks_cosine_rf_destroy releases it.  Maps gathered into one feature source must be of one kind. */
KS_API int32_t ks_padded_fft_create(int64_t ctx, const double* signs_or_null, int64_t n_in, int32_t rectify, double max_val,
                                    double alpha, int64_t* out_rf);
/* Elementwise nodes on a materialised batch: op 0: out = x .* colvec (RandomSignNode.apply), op 1: out = max(a, x - b)
 * (LinearRectifier.apply); returns a new matrix. */
KS_API int32_t ks_matrix_map(int64_t ctx, int64_t m, int32_t op, const double* colvec_or_null, double a, double b, int64_t* out_m);

/* ---- Convolver [andThen SymmetricRectifier andThen Pooler(sum) andThen ImageVectorizer] ---------------------------------
 * The featurizer of K/pipelines/images/cifar/RandomPatchCifar.scala:59-63 (K/nodes/images/Convolver.scala:20-203,
 * SymmetricRectifier.scala:7-32, Pooler.scala:21-69, K/utils/Stats.scala:112-123).  filters: DenseMatrix (n_filters x
 * conv_size^2*channels) column-major, columns ordered c + x*channels + y*channels*conv_size (Convolver.packFilters), already whitened
 * if a whitener is used; whitener_means (patch dimension) may be NULL.  Images are rows of a matrix in ImageVectorizer order
 * (value (x, y, c) at c + x*channels + y*channels*x_dim; x_dim = image height, K/utils/images/Image.scala:140-143).
 * ks_convolver_apply with pool_size = 0 returns the convolved images (n x resW*resH*n_filters, same vectorised order);
 * with pool_size > 0 the rectifier and the sum pooling run in the GEMM's epilogue and only the pooled features
 * (n x nPoolsX*nPoolsY*2*n_filters) are written. */
KS_API int32_t ks_convolver_create(int64_t ctx, const double* filters_colmajor, int32_t n_filters, int32_t x_dim, int32_t y_dim,
                                   int32_t channels, int32_t conv_size, const double* whitener_means_or_null, int32_t normalize_patches,
                                   double var_constant, int64_t* out_conv);
KS_API int32_t ks_convolver_apply(int64_t ctx, int64_t conv, int64_t images, int32_t pool_stride, int32_t pool_size, double max_val,
                                  double alpha, int64_t* out_features);
KS_API int32_t ks_convolver_destroy(int64_t ctx, int64_t conv);

/* ---- feature source shared by fit / apply -------------------------------------------------
 * Either `features` (a materialised N x D matrix; VectorSplitter blocks are column ranges of it,
 * K/nodes/util/VectorSplitter.scala:15-25) or `x_in` + `rfs[n_rfs]` (the gather of
 * CosineRandomFeatures nodes followed by VectorCombiner, K/pipelines/speech/TimitPipeline.scala:76-93),
 * whose feature blocks are regenerated on the fly and never stored.  Pass 0 for the unused one. */

/* BlockLeastSquaresEstimator(blockSize, numIter, lambda, numFeaturesOpt).fit(features, labels)
 * (K/nodes/learning/BlockLinearMapper.scala:199-257).  Collective across ranks. */
KS_API int32_t ks_blockls_fit(int64_t ctx, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int64_t labels,
                       int32_t block_size, int32_t num_iter, double lambda, int64_t num_features_or_0,
                       int32_t precision_mode, int64_t* out_model);
/* BlockWeightedLeastSquaresEstimator(blockSize, numIter, lambda, mixtureWeight, numFeaturesOpt).fit
 * (K/nodes/learning/BlockWeightedLeastSquares.scala:36-84, trainWithL2 :102-321).  Rows need not be
 * class-sorted within a rank (groupByClasses :333-370 is applied on the device).  With world_size > 1 the rows must be
 * sharded BY CLASS: every class lives on exactly one rank (checked; KS_ERR_INVALID otherwise).  Collective across ranks. */
KS_API int32_t ks_blockwls_fit(int64_t ctx, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int64_t labels,
                        int32_t block_size, int32_t num_iter, double lambda, double mixture_weight,
                        int64_t num_features_or_0, int32_t precision_mode, int64_t* out_model);
/* LinearMapEstimator(lambda).fit (K/nodes/learning/LinearMapper.scala:69-98): exact centred normal
 * equations == one block covering all features.  has_lambda = 0 mirrors lambda = None. */
KS_API int32_t ks_linear_map_fit(int64_t ctx, int64_t features, int64_t labels, int32_t has_lambda, double lambda,
                          int64_t* out_model);
/* DenseLBFGSwithL2(LeastSquaresDenseGradient, fitIntercept, numCorrections, convergenceTol, numIterations, regParam).fit
 * (K/nodes/learning/LBFGS.scala:135-173): minimises |A_c W - Y_c|^2 / (2N) + reg_param / 2 |W|^2 from W = 0 by L-BFGS with the
 * last num_corrections pairs and the exact step along each direction (DESIGN.md section 14).  fit_intercept != 0 centres
 * features and labels by their exact means and returns LinearMapper(W, label mean, feature means); 0 returns W alone.  Stops
 * after num_iterations steps or, with convergence_tol > 0, when the loss or the gradient has converged; ks_last_fit_stats_json
 * reports iterations, loss_history (f(W_0) .. f(W_T)) and stop_reason.  num_corrections and num_iterations must be >= 1,
 * reg_param and convergence_tol finite and >= 0.  Returns an ordinary model handle.  Collective across ranks. */
KS_API int32_t ks_lbfgs_fit(int64_t ctx, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int64_t labels,
                            int32_t fit_intercept, int32_t num_corrections, double convergence_tol, int32_t num_iterations,
                            double reg_param, int32_t precision_mode, int64_t* out_model);

/* ---- BlockLinearMapper / LinearMapper state (K/nodes/learning/BlockLinearMapper.scala:22-33,
 * K/nodes/learning/LinearMapper.scala:18-22) ------------------------------------------------ */
KS_API int32_t ks_model_from_host(int64_t ctx, const double* const* xs_colmajor, const int64_t* block_rows, int32_t n_blocks,
                           int64_t k, const double* b_or_null, const double* const* feature_means_or_null,
                           int32_t block_size, int64_t* out_model);
KS_API int32_t ks_model_num_blocks(int64_t ctx, int64_t model, int32_t* n_blocks, int64_t* k, int32_t* block_size);
KS_API int32_t ks_model_block_rows(int64_t ctx, int64_t model, int32_t j, int64_t* rows);
/* W_j as a column-major (rows_j x k) fp64 matrix; mean_out (rows_j) may be NULL; *has_mean tells whether the
 * model carries feature scalers (BlockLS: yes, BWLS: no -- BlockWeightedLeastSquares.scala:316-320). */
KS_API int32_t ks_model_get_block(int64_t ctx, int64_t model, int32_t j, double* W_colmajor_out, double* mean_out,
                           int32_t* has_mean);
KS_API int32_t ks_model_get_intercept(int64_t ctx, int64_t model, double* b_out, int32_t* has_intercept);
/* Zero-copy access to the model's pinned host mirror (written by async device-to-host copies while the fit was still running):
 * *W_ptr = block j, column-major rows_j x k; *mean_ptr = rows_j means or NULL; *intercept_ptr = k values or NULL.  The pointers
 * stay valid until ks_model_destroy.  Any argument may be NULL.  (A JNI caller hands them to SetDoubleArrayRegion.) */
KS_API int32_t ks_model_host_view(int64_t ctx, int64_t model, int32_t j, const double** W_ptr, const double** mean_ptr,
                                  const double** intercept_ptr);
/* Fitted model <-> flat little-endian file ("KSB2MDL1", int32 block_size, int32 n_blocks, int64 k, int32 has_mean,
 * int32 has_intercept, int64 rows[n_blocks], per block W (rows x k fp64 column-major) [+ rows means], k intercepts): replaces
 * the Java-serialised FittedPipeline for the BlockLinearMapper stage (K/workflow/FittedPipeline.scala:18-22). */
KS_API int32_t ks_model_save(int64_t ctx, int64_t model, const char* path);
KS_API int32_t ks_model_load(int64_t ctx, const char* path, int64_t* out_model);
/* BlockLinearMapper.apply(RDD) :40-73 -> new (N x k) matrix of predictions. */
KS_API int32_t ks_model_apply(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs,
                       int64_t* out_predictions);
/* apply followed by MaxClassifier (K/nodes/util/MaxClassifier.scala:9-11); host_out has N int32. */
KS_API int32_t ks_model_apply_argmax(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs,
                              int32_t n_rfs, int32_t* host_out);
/* applyAndEvaluate (BlockLinearMapper.scala:95-137): the cumulative prediction after block j (intercept included). */
KS_API int32_t ks_model_apply_partial(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs,
                               int32_t n_rfs, int32_t last_block, int64_t* out_predictions);
/* apply -> MaxClassifier on predictions and on the +-1 indicator labels -> confusion matrix (K/evaluation/MulticlassClassifierEvaluator.scala:130-161), all on the device,
   summed over the ranks; out_counts is k x k row-major, rows = true class, columns = predicted class.  Collective. */
KS_API int32_t ks_model_confusion_matrix(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs,
                                         int32_t n_rfs, int64_t labels, double* out_counts);
/* BlockLeastSquaresEstimator.computeCost (K/nodes/learning/BlockLinearMapper.scala:142-187); collective. */
KS_API int32_t ks_model_cost(int64_t ctx, int64_t model, int64_t features, int64_t x_in, const int64_t* rfs, int32_t n_rfs,
                      int64_t labels, double lambda, double* out_cost);
KS_API int32_t ks_model_destroy(int64_t ctx, int64_t model);

/* ---- Gaussian-kernel ridge regression -------------------------------------------------------
 * GaussianKernelGenerator(gamma).fit(train) (K/nodes/learning/KernelGenerator.scala:121-176): K(x, y) = exp(-gamma |x - y|^2).
 * Collective: every rank passes its training rows; the kernel object holds ALL training rows on every rank (gathered in rank
 * order: the global row order of the fit and of the model blocks), shifted by their exact fp64 column mean.
 * gamma must be finite and > 0. */
KS_API int32_t ks_gaussian_kernel_create(int64_t ctx, int64_t x_train, double gamma, int64_t* out_kernel);
/* KernelMatrix(colIdxs) (K/nodes/learning/KernelMatrix.scala): K(x, x_train[col0, col0 + cols)) as a new (x rows x cols) fp32
 * matrix; x holds raw input rows with the training column count. */
KS_API int32_t ks_gaussian_kernel_block(int64_t ctx, int64_t kernel, int64_t x, int64_t col0, int64_t cols, int64_t* out_m);
/* training rows over all ranks (the columns of the kernel matrix) and their width; either pointer may be NULL */
KS_API int32_t ks_gaussian_kernel_shape(int64_t ctx, int64_t kernel, int64_t* n_train, int64_t* dim);
KS_API int32_t ks_gaussian_kernel_destroy(int64_t ctx, int64_t kernel);
/* KernelRidgeRegression(kernelGenerator, lambda, blockSize, numEpochs, blockPermuter).fit (K/nodes/learning/
 * KernelRidgeRegression.scala:116-200): block Gauss-Seidel on (K + lambda I) W = Y over contiguous blocks of training rows, no
 * centring, no intercept.  labels: this rank's rows.  block_order (num_epochs x n_blocks, each row a permutation of the blocks)
 * or NULL for the sequential order.  Returns a kernel model (KernelBlockLinearMapper): ks_model_apply / _apply_argmax /
 * _confusion_matrix take the raw input rows as `features` (x_in = 0, no rfs); ks_model_save / _cost / _apply_partial reject it.
 * K_BB + lambda I not positive definite (lambda = 0 with repeated rows): KS_ERR_NOT_SPD on every rank.  Collective. */
KS_API int32_t ks_krr_fit(int64_t ctx, int64_t kernel, int64_t labels, double lambda, int32_t block_size, int32_t num_epochs,
                          const int32_t* block_order_or_null, int64_t* out_model);
/* new KernelBlockLinearMapper(xs, blockSize, kernelTransformer, nTrain): block_rows must sum to the kernel's training rows. */
KS_API int32_t ks_kernel_model_from_host(int64_t ctx, int64_t kernel, const double* const* xs_colmajor, const int64_t* block_rows,
                                         int32_t n_blocks, int64_t k, int32_t block_size, int64_t* out_model);

/* ---- on-disk formats at the edges of the path (host code; need no context) -----------------
 * Headerless CSV of doubles (K/loaders/CsvDataLoader.scala:28-30): ks_csv_dims counts rows and the fields of the first row;
 * ks_csv_read_* parse into a caller-owned row-major buffer (pinned memory makes the following upload asynchronous), split by
 * lines over the host threads.  MNIST CSVs carry the 1-based label in column 0 (K/pipelines/images/mnist/MnistRandomFFT.scala:34-36). */
KS_API const char* ks_io_last_error(void);
KS_API int32_t ks_csv_dims(const char* path, int64_t* n_rows, int64_t* n_cols);
KS_API int32_t ks_csv_read_f64(const char* path, double* out, int64_t n_rows, int64_t n_cols, int64_t ld);
KS_API int32_t ks_csv_read_f32(const char* path, float* out, int64_t n_rows, int64_t n_cols, int64_t ld);
/* TIMIT sparse label file, lines "row label", both 1-based (K/loaders/TimitFeaturesDataLoader.scala:22-42):
 * labels_out[row - 1] = label - 1; rows the file does not mention keep -1. */
KS_API int32_t ks_timit_labels_read(const char* path, int32_t* labels_out, int64_t n_rows);
/* CIFAR-10 binary records, 1 label byte + 3072 image bytes (K/loaders/CifarLoader.scala:30-45).  With both output pointers NULL
 * only *n_out (the record count) is set. */
KS_API int32_t ks_cifar_read(const char* path, uint8_t* images_out, int32_t* labels_out, int64_t max_records, int64_t* n_out);

/* ---- instrumentation ----------------------------------------------------------------------
 * JSON with per-phase device milliseconds of the last fit (featurize, gram, allreduce, solve, update),
 * kernel launch count and the algorithmic flop count. */
KS_API int32_t ks_last_fit_stats_json(int64_t ctx, char* buf, int64_t buflen);
/* bytes ks_last_fit_stats_json needs for the current JSON, terminating NUL included */
KS_API int32_t ks_last_fit_stats_json_size(int64_t ctx, int64_t* out_bytes);
/* number of kernels this library has launched on the context since creation */
KS_API int32_t ks_ctx_launch_count(int64_t ctx, int64_t* out_count);

/* ---- low-level kernel entry points (unit tests and micro-benchmarks) ----------------------- */
/* out_g (M x M, row-major fp64, ld_g) = A^T A upper triangle mirrored; out_c (M x Nb) = A^T B; A, B device matrices
 * with equal row counts.  Exercises the Gram kernel alone (no centring, no collective). */
KS_API int32_t ks_debug_gram(int64_t ctx, int64_t a, int64_t b, double* out_g, int64_t ld_g, double* out_c, int64_t ld_c);
/* Times `iters` launches of the Gram kernel alone (CUDA events on the launching stream); returns ms per launch. */
KS_API int32_t ks_debug_time_gram(int64_t ctx, int64_t a, int64_t b, int32_t iters, double* out_ms);

/* X = H^-1 B for a symmetric positive definite H (column-major n x n) and B (column-major n x k): Cholesky with cuSOLVER, then
 * either the library's own multi-RHS solve kernel (use_cusolver = 0; option "custom_solve") or cusolverDnDpotrs (the default of
 * the fits); best-of-3 ms. */
KS_API int32_t ks_debug_chol_solve(int64_t ctx, const double* H_colmajor, int32_t n, const double* B_colmajor, int32_t k,
                                   int32_t use_cusolver, double* X_out, double* out_ms);

#ifdef __cplusplus
}
#endif
#endif /* KEYSTONE_B200_H */
