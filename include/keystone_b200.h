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
 * right-hand-side columns over the ranks], "reserve_sms" [8], "host_mirror" [1: fits copy each finished model block into pinned host memory while they run]; "custom_solve" [-1: automatic -- the library's own DMMA
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
 * (LinearRectifier.apply), op 2: out = sign(x) sqrt(|x|) ((Batch)SignedHellingerMapper, K/nodes/stats/SignedHellingerMapper.scala;
 * colvec, a and b unused); returns a new matrix. */
KS_API int32_t ks_matrix_map(int64_t ctx, int64_t m, int32_t op, const double* colvec_or_null, double a, double b, int64_t* out_m);
/* NormalizeRows (K/nodes/stats/NormalizeRows.scala): every row divided by max(|row|_2, 2.2e-16), the norm in fp64; a new matrix. */
KS_API int32_t ks_matrix_normalize_rows(int64_t ctx, int64_t m, int64_t* out_m);

/* ---- LCS descriptors, GMM posteriors, Fisher vectors (DESIGN.md section 16) -------------------------------------------------
 * The LCS branch of K/pipelines/images/imagenet/ImageNetSiftLcsFV.scala.  Item batches (the reference's one DenseMatrix per image)
 * are one device matrix with one descriptor per ROW plus item row offsets.  None of these is collective: each rank encodes its
 * own images. */
/* LCSExtractor(stride, strideStart, subPatchSize).apply (K/nodes/images/LCSExtractor.scala) on a batch of equal-size images, rows of
 * `images` in ImageVectorizer order (value (x, y, c) at c + x*channels + y*channels*x_dim, x_dim = image height).  Window means and
 * standard deviations in fp64, rounded once to fp32.  Output: (n_images * nKP) x (n^2 * channels * 2); image i owns rows
 * [i nKP, (i+1) nKP), keypoint (xk, yk) is row xk * numPoolsY + yk, column ((c * n + nx) * n + ny) * 2 + {0: mean, 1: std}.
 * Rejects bad shapes, no keypoint, and neighbourhoods that leave the image. */
KS_API int32_t ks_lcs_extract(int64_t ctx, int64_t images, int32_t x_dim, int32_t y_dim, int32_t channels, int32_t stride,
                              int32_t stride_start, int32_t sub_patch_size, int64_t* out_m);
/* GaussianMixtureModel(means, variances, weights, weightThreshold) (K/nodes/learning/GaussianMixtureModel.scala): means and variances
 * dim x k column-major (Breeze), k weights.  Rejects non-finite values, variances <= 0, weights <= 0, dim > 1024 and a threshold
 * outside [0, 1/k). */
KS_API int32_t ks_gmm_create(int64_t ctx, const double* means_colmajor, const double* variances_colmajor, const double* weights,
                             int64_t dim, int64_t k, double weight_threshold, int64_t* out_gmm);
KS_API int32_t ks_gmm_destroy(int64_t ctx, int64_t gmm);
/* GaussianMixtureModel.apply(X): x (N x dim) -> N x k thresholded posteriors, computed in fp64 and stored as fp32. */
KS_API int32_t ks_gmm_posteriors(int64_t ctx, int64_t gmm, int64_t x, int64_t* out_m);
/* FisherVector(gmm).apply andThen MatrixVectorizer (K/nodes/images/FisherVector.scala) for every item: descriptors (rows x dim), item
 * i = rows [item_offsets[i], item_offsets[i+1]) (n_items + 1 host offsets, 0 first, rows last, strictly increasing).  Output
 * n_items x (2 dim k) fp32, element (d, j) of the dim x 2k matrix [fv1 | fv2] at column d + dim * j.  Statistics in fp64 on the DMMA
 * tensor core, in a fixed order (bit-reproducible); fv2 is the Sanchez et al. formula (DESIGN.md section 16). */
KS_API int32_t ks_fisher_vector_apply(int64_t ctx, int64_t gmm, int64_t descriptors, const int64_t* item_offsets, int64_t n_items,
                                      int64_t* out_m);

/* ---- Gaussian-mixture EM and k-means++ (DESIGN.md section 17) ---------------------------------------------------------------
 * The fits of K/nodes/learning/{GaussianMixtureModelEstimator,KMeansPlusPlus}.scala on the rows of x (N x dim), in fp64 on the
 * device, without float atomics (a repeated fit returns identical bits).  Not collective: each rank fits on the rows it is given.
 * Every fit writes ks_last_fit_stats_json: solver ("gmm" / "kmeans"), n, d, k, iterations, stop_reason ("max_iterations", "cost",
 * "min_cluster_size"), cost_history, seed_rows, seeding / init / estep / stats / mstep milliseconds and launches.
 * Rejected with KS_ERR_INVALID: k <= 0, N < k, dim > 1024, non-finite input, uniforms outside [0, 1), and fewer distinct points than
 * centres; a cluster the k-means passes leave empty is an error that names it (the reference divides by zero there).
 *
 * Randomness: the reference's MersenneTwister / Multinomial stream is not reproduced; the caller passes the uniforms.  k-means++
 * takes num_means uniforms u_j in [0, 1):
 *   centre 0 is row min(floor(u_0 N), N - 1);
 *   after centre j - 1, every row holds d_n = min over the centres so far of 1/2 sum_d (x_nd - c_d)^2 (fp64, the sum over d in
 *   order, no fused multiply-add).  Blocks are the rows [256 b, 256 b + 256); B_b = the tree sum of the block's d (pairs at
 *   distance 128, 64, ..., 1, zeros past N); P_b = B_0 + ... + B_(b-1) and W = P_nblocks, summed left to right.  W = 0: error.
 *   Centre j is in the first block with P_b + B_b > u_j W (none: the last block with B_b > 0), at the first row n of that block with
 *   P_b + s_n > u_j W, s_n the inclusive prefix sum of d over the block's rows in order (none: the block's last row with d_n > 0). */
/* KMeansPlusPlusEstimator(num_means, max_iterations, stop_tolerance).fit(x): the seeding above, then up to max_iterations Lloyd
 * passes (assignment to the first nearest centre, cost = mean best distance, means = sums / counts; stop after the pass whose
 * cost fails (prev - cur) >= stop_tolerance |prev|).  means_out: num_means x dim row-major; seed_rows_or_null: the num_means
 * seed rows. */
KS_API int32_t ks_kmeans_fit(int64_t ctx, int64_t x, int64_t num_means, int32_t max_iterations, double stop_tolerance,
                             const double* uniforms, double* means_out, int64_t* seed_rows_or_null, int32_t* iterations_or_null);
/* KMeansModel(means).apply(x): the N x num_means one-hot assignment (fp32) to the first nearest of the means (num_means x dim,
 * row-major). */
KS_API int32_t ks_kmeans_assign(int64_t ctx, int64_t x, const double* means_rowmajor, int64_t num_means, int64_t dim, int64_t* out_m);
/* GaussianMixtureModelEstimator(k, maxIterations, minClusterSize, stopTolerance, weightThreshold, smallVarianceThreshold,
 * absoluteVarianceThreshold, initializationMethod).fit(x).  initialization 0: k-means++ (uniforms: k values, the rule above; one
 * Lloyd pass, then weights, means and variances of the hard assignment to the updated means); 1: random (uniforms: k x dim
 * row-major, means = colMin + u range, variances = 0.1 range^2, weights 1/k).  Variances are floored at
 * max(smallVarianceThreshold varGlobal_d, absoluteVarianceThreshold).  EM stops when (cur - prev) < stopTolerance |prev| (from the
 * second iteration; that E-step counts as an iteration, no M-step follows), or when a component's posterior mass is below
 * minClusterSize (the previous parameters are kept).  weightThreshold must lie in [0, 1/k); absoluteVarianceThreshold must be > 0.
 * Returns a model handle with weightThreshold 1e-4 (as the reference's GaussianMixtureModel(means, vars, weights)), its means and
 * variances (dim x k column-major), k weights and the number of E-steps evaluated. */
KS_API int32_t ks_gmm_fit(int64_t ctx, int64_t x, int64_t k, int32_t max_iterations, double min_cluster_size, double stop_tolerance,
                          double weight_threshold, double small_variance_threshold, double absolute_variance_threshold,
                          int32_t initialization, const double* uniforms, int64_t* out_gmm, double* means_colmajor_out,
                          double* variances_colmajor_out, double* weights_out, int32_t* iterations_or_null);
/* out = rows rows[0..n) of m, in that order, as a new matrix (ColumnSampler on an item batch); indices must lie in [0, rows). */
KS_API int32_t ks_matrix_gather_rows(int64_t ctx, int64_t m, const int64_t* rows, int64_t n, int64_t* out_m);

/* ---- PixelScaler, GrayScaler and dense multi-scale SIFT (DESIGN.md section 18) -----------------------------------------------
 * The first three nodes of K/pipelines/images/voc/VOCSIFTFisher.scala and of the SIFT half of ImageNetSiftLcsFV.scala.  Images are
 * rows in ImageVectorizer order (value (x, y, c) at c + x*channels + y*channels*x_dim, x_dim = image height), all of one shape.
 * Non-finite pixels are rejected with KS_ERR_INVALID.  None of these is collective. */
/* PixelScaler (K/nodes/images/PixelScaler.scala): every value / 255.0 in fp64, rounded once to fp32; a new matrix. */
KS_API int32_t ks_image_pixel_scale(int64_t ctx, int64_t images, int64_t* out_m);
/* GrayScaler (ImageUtils.toGrayScale), after PixelScaler when pixel_scale is 1: in fp64, 0.2989 R + 0.5870 G + 0.1140 B with B at
 * channel 0 for three channels, sqrt(sum_c v^2 / channels) otherwise; rounded once to fp32.  Output: one-channel images,
 * n_images x (x_dim * y_dim).  Rejects bad shapes and pixel_scale outside {0, 1}. */
KS_API int32_t ks_image_grayscale(int64_t ctx, int64_t images, int32_t x_dim, int32_t y_dim, int32_t channels, int32_t pixel_scale,
                                  int64_t* out_m);
/* SIFTExtractor(step, bin, scales, scale_step).apply (K/nodes/images/external/SIFTExtractor.scala) on one-channel images
 * (n_images x (x_dim * y_dim)): vlfeat's dense SIFT with a flat window at every scale s < scales (bin + 2s, step + s*scale_step),
 * the contrast threshold 0.005 and the reference's transposed uint8 quantisation.  Output: (n_images * nKP) x 128 fp32 holding
 * integers in [0, 255], one descriptor per ROW (the reference's columns); image i owns rows [i nKP, (i+1) nKP), scales follow in
 * order, and within a scale frames run along y outer, x inner, as vlfeat (which sees the image transposed) emits them.  A scale
 * without frames contributes no rows.  Rejects bad shapes, step < 1, bin < 1, scales < 1, scale_step < 0 and oversized
 * parameters (step, scale_step > 65536, bin > 4096, scales > 256). */
KS_API int32_t ks_sift_extract(int64_t ctx, int64_t gray_images, int32_t x_dim, int32_t y_dim, int32_t step, int32_t bin, int32_t scales,
                               int32_t scale_step, int64_t* out_m);
/* Host only: counts_out[s] (scales entries) = the keypoints ks_sift_extract emits per image at scale s.  Returns KS_ERR_INVALID
 * for the arguments ks_sift_extract rejects. */
KS_API int32_t ks_sift_keypoints(int32_t x_dim, int32_t y_dim, int32_t step, int32_t bin, int32_t scales, int32_t scale_step,
                                 int64_t* counts_out);

/* ---- HOG and DAISY descriptors (DESIGN.md section 19) --------------------------------------------------------------------------
 * Images as for SIFT above: rows in ImageVectorizer order, all of one shape; image i owns a contiguous row range of the output, and
 * an image with no cell or keypoint contributes no rows.  Non-finite pixels are rejected with KS_ERR_INVALID.  Not collective. */
/* HogExtractor(bin).apply (K/nodes/images/HogExtractor.scala) on three-channel BGR images, after PixelScaler when pixel_scale is 1
 * (x / 255.0 in fp64, never rounded).  nX = round(x_dim / bin), nY = round(y_dim / bin) cells; output (n_images * (nX-2)(nY-2)) x 32
 * fp32, the reference's cells x 32 matrix per image with row y + x (nY - 2): 18 contrast-sensitive, 9 contrast-insensitive and 4
 * texture values and a zero.  Reads past the visible edge are the reference's unclamped reads of c + x*3 + y*3*x_dim; rejects bin
 * and shape pairs where such a read passes the end of the image, channels != 3, bin outside [1, 1024], bad shapes and pixel_scale
 * outside {0, 1}. */
KS_API int32_t ks_hog_extract(int64_t ctx, int64_t images, int32_t x_dim, int32_t y_dim, int32_t channels, int32_t pixel_scale, int32_t bin,
                              int64_t* out_m);
/* DaisyExtractor(T, Q, R, H, border, stride).apply (K/nodes/images/DaisyExtractor.scala) on one-channel images: gradients, H
 * rectified orientation maps and Q Gaussian blur layers in fp64 (ImageUtils.conv2D), keypoints x = border .. x_dim-border-1 by
 * stride outer, y likewise inner.  Output: (n_images * nKP) x (H (T Q + 1)) fp32, one keypoint per ROW (the reference's columns):
 * the centre histogram at columns [0, H), ring sample (l, t) at H + t Q H + l H, each normalised to unit L2 norm or zeroed when its
 * norm is <= 1e-8.  Rejects T, Q, R, H, stride < 1, border < 0, oversized parameters (T, H > 64, Q > 16, R > 4096, a blur radius
 * > 1024, stride or border > 65536), ring samples that leave the image and bad shapes. */
KS_API int32_t ks_daisy_extract(int64_t ctx, int64_t gray_images, int32_t x_dim, int32_t y_dim, int32_t T, int32_t Q, int32_t R, int32_t H,
                                int32_t border, int32_t stride, int64_t* out_m);

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
/* The same chain over views of src_x x src_y source images (views as for ks_image_views, each of the Convolver's x_dim x y_dim):
 * equal to ks_convolver_apply on ks_image_views' output, without materialising it (each image chunk's views are gathered into a
 * staging buffer).  Unpooled output is bit-identical to that; pooled output, like ks_convolver_apply's, adds the pool sums with fp32
 * atomics, so it agrees to the rounding of that order. */
KS_API int32_t ks_convolver_apply_views(int64_t ctx, int64_t conv, int64_t images, int32_t src_x, int32_t src_y, const int32_t* views,
                                        int64_t n_views, int32_t pool_stride, int32_t pool_size, double max_val, double alpha,
                                        int64_t* out_features);

/* ---- image views, Stats.normalizeRows, StandardScaler, AugmentedExamplesEvaluator (DESIGN.md section 21) -----------------------
 * The front end and the test-time augmentation of K/pipelines/images/cifar/RandomPatchCifar{,Augmented}.scala.  Only the scaler fit
 * is collective. */
/* Windower, Cropper, RandomPatcher, CenterCornerPatcher and RandomImageTransformer(flipHorizontal) as a table of views of a batch of
 * x_dim x y_dim x channels images (rows in ImageVectorizer order): views is n_views x 4 int32 (src_row, x0, y0, flip).  Output
 * n_views x (out_x out_y channels), view v holding ImageUtils.crop(src, x0, y0, x0 + out_x, y0 + out_y), reversed along y
 * (ImageUtils.flipHorizontal) when flip is 1, as exact copies.  KS_ERR_INVALID: a view crop would reject (outside the image), a
 * src_row outside the batch, flip outside {0, 1}, out_x or out_y < 1. */
KS_API int32_t ks_image_views(int64_t ctx, int64_t images, int32_t x_dim, int32_t y_dim, int32_t channels, const int32_t* views, int64_t n_views,
                              int32_t out_x, int32_t out_y, int64_t* out_m);
/* Stats.normalizeRows(mat, alpha) (K/utils/Stats.scala:112-123): per row, subtract the mean (NaN -> 0) and divide by
 * sqrt(sample variance + alpha) (NaN -> sqrt(alpha)), in fp64, rounded once to fp32; a new matrix.  alpha must be finite.  (The
 * L2 NormalizeRows node is ks_matrix_normalize_rows.) */
KS_API int32_t ks_matrix_stats_normalize_rows(int64_t ctx, int64_t m, double alpha, int64_t* out_m);
/* StandardScaler(normalizeStdDev, eps).fit (K/nodes/stats/StandardScaler.scala:38-59): fp64 column means of x over all ranks and,
 * with normalize_std = 1, the unbiased column std (0 for one row), replaced by 1.0 where it is NaN, infinite or below eps.
 * mean_out / std_out: cols values each (std_out unused when normalize_std = 0).  Column sums run over fixed row chunks added in
 * order, without float atomics: a refit on the same rows returns identical bits.  KS_ERR_INVALID: no rows on any rank, eps not
 * finite or < 0, normalize_std outside {0, 1}.  Collective. */
KS_API int32_t ks_standard_scaler_fit(int64_t ctx, int64_t x, int32_t normalize_std, double eps, double* mean_out, double* std_out);
/* StandardScalerModel(mean, std).apply: (x - mean) [/ std] in fp64, rounded once to fp32; a new matrix, padding columns zero.
 * KS_ERR_INVALID for a non-finite mean or a std that is zero or not finite. */
KS_API int32_t ks_standard_scaler_apply(int64_t ctx, int64_t x, const double* mean, const double* std_or_null, int64_t* out_m);
/* AugmentedExamplesEvaluator(names, numClasses, policy).evaluate (K/evaluation/AugmentedExamplesEvaluator.scala) on this rank's
 * score rows (n_views x k, BlockLinearMapper.apply's output): group g is the views rows[group_offsets[g] .. group_offsets[g+1]),
 * added in that order in fp64 -- policy 0 (average) the scores, divided by the count; policy 1 (borda) each class's rank in the
 * view's ascending stable sort.  Then the first maximum is the prediction.  labels: n_views class ids indexed by score row.
 * out_counts: k x k row-major (rows = true class, columns = prediction), as ks_model_confusion_matrix.  KS_ERR_INVALID: rows not a
 * permutation of the score rows, offsets not strictly increasing from 0 to n_views, a label outside [0, k), views of one group
 * with different labels, k != the score columns or k > 4096.  Not collective. */
KS_API int32_t ks_grouped_confusion_matrix(int64_t ctx, int64_t scores, const int64_t* rows, const int64_t* group_offsets, int64_t n_groups,
                                           const int32_t* labels, int64_t k, int32_t policy, double* out_counts);

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

/* ---- sparse matrices and SparseLBFGSwithL2 (DESIGN.md section 20) ---------------------------------------------------------------
 * A rank's rows of a row-sharded sparse matrix (the reference's RDD[SparseVector[Double]], K/nodes/learning/LBFGS.scala:208-281).
 * Sparse handles are typed: passing one where a dense matrix handle is expected, or the reverse, returns KS_ERR_HANDLE. */
/* CSR upload of this rank's n_rows rows: indptr (n_rows + 1), indices and values (indptr[n_rows] each), borrowed for the call.
 * Stored as fp64 values, int32 column indices and int64 offsets, plus a CSC copy of the same entries built on the device (a stable
 * radix sort: rows ascend within a column) and work tables that cut long rows and columns into chunks of bounded length.
 * Unsorted indices within a row and repeated (row, column) entries are legal; every entry contributes its own product, so repeated
 * entries add up (Breeze's SparseVector built with repeated keys).  Empty rows and n_rows = 0 are legal.  KS_ERR_INVALID with a
 * message: indptr[0] != 0, a decreasing indptr, an index outside [0, n_cols), a non-finite value, n_cols outside [1, INT32_MAX],
 * n_rows outside [0, INT32_MAX]. */
KS_API int32_t ks_sparse_from_host_csr(int64_t ctx, const int64_t* indptr, const int32_t* indices, const double* values, int64_t n_rows,
                                       int64_t n_cols, int64_t* out_s);
KS_API int32_t ks_sparse_shape(int64_t ctx, int64_t s, int64_t* n_rows, int64_t* n_cols, int64_t* nnz);
/* The CSR of s as stored (rows + 1 offsets, nnz column indices and values) into caller buffers. */
KS_API int32_t ks_sparse_to_host_csr(int64_t ctx, int64_t s, int64_t* indptr, int32_t* indices, double* values);
KS_API int32_t ks_sparse_destroy(int64_t ctx, int64_t s);
/* Densify (K/nodes/util/Densify.scala): a new n_rows x n_cols fp32 matrix; repeated entries are summed in fp64 in upload order and
 * rounded once. */
KS_API int32_t ks_sparse_densify(int64_t ctx, int64_t s, int64_t* out_m);
/* SparseLBFGSwithL2(LeastSquaresSparseGradient, fitIntercept, numCorrections, convergenceTol, numIterations, regParam).fit
 * (K/nodes/learning/LBFGS.scala:208-262): no centring; with fit_intercept the data gets an implicit column of ones, and the fit
 * minimises f = |[A 1][W; b] - Y|^2 / (2N) + reg_param / 2 |[W; b]|^2 (the bias is regularised in f and in g) from zero by the
 * recursion, exact step and stop rules of ks_lbfgs_fit, all in fp64; labels are the fp32 matrix of this rank's rows.  Returns an
 * ordinary model handle, W in feature blocks of min(d, 4096) rows, b as the intercept (fit_intercept = 0: W alone), no feature
 * means.  Both products are gathers in a fixed summation order: one rank fitting the same input twice gets bit-identical models,
 * and every rank ends with the same bits.  ks_last_fit_stats_json adds solver "sparse_lbfgs" and the global nnz.  Collective. */
KS_API int32_t ks_sparse_lbfgs_fit(int64_t ctx, int64_t s, int64_t labels, int32_t fit_intercept, int32_t num_corrections,
                                   double convergence_tol, int32_t num_iterations, double reg_param, int64_t* out_model);
/* SparseLinearMapper.apply (K/nodes/learning/SparseLinearMapper.scala): A W + b over the CSR rows of s in fp64, rounded once into a
 * new N x k fp32 matrix.  KS_ERR_INVALID for a model with feature means, a kernel model, or n_cols != the model's d. */
KS_API int32_t ks_model_apply_sparse(int64_t ctx, int64_t model, int64_t s, int64_t* out_predictions);

/* ---- logistic regression and multinomial naive Bayes (DESIGN.md section 22) ---------------------------------------------------
 * Both take this rank's rows from exactly one feature source -- a dense fp32 matrix handle (features_or_0) or a sparse handle
 * (sparse_or_0), the other 0 -- and labels: n_labels class ids in [0, num_classes) on the host (n_labels = the rank's rows,
 * num_classes >= 2).  A label outside the range on any rank (and, for naive Bayes, a negative or NaN feature value or a class with no
 * rows over all ranks) is flagged, all-reduced and rejected on every rank with KS_ERR_INVALID.  Every sum has a fixed order: one rank
 * fitting the same input twice gets a bit-identical model, and every rank ends with the same bits.  Both are collective and return an
 * ordinary model handle (d x k in feature blocks of min(d, 4096) rows, no feature means). */
/* LogisticRegressionEstimator(numClasses, regParam, numIters, convergenceTol).fit (K/nodes/learning/LogisticRegressionModel.scala,
 * MLlib's LogisticGradient + SquaredL2Updater): minimises (1/N) sum_i [lse(0, Z_i) - Z_{i,y_i}] + reg_param / 2 |W|^2 over W
 * (d x (k-1), Z = A W, class 0 the pivot) from W = 0 by L-BFGS (10 corrections, the stop rules of ks_lbfgs_fit) with a strong-Wolfe
 * line search in fp64.  The model's column 0 is zero and it has no intercept, so ks_model_apply_argmax is MLlib's predict.
 * ks_last_fit_stats_json: solver "logistic_regression", iterations, loss_history, stop_reason (also "line_search_failed"),
 * line_search_evals (trials per line search), per-phase device ms.  num_iterations >= 1, reg_param and convergence_tol finite, >= 0. */
KS_API int32_t ks_logistic_fit(int64_t ctx, int64_t features_or_0, int64_t sparse_or_0, const int32_t* labels, int64_t n_labels,
                               int32_t num_classes, double reg_param, int32_t num_iterations, double convergence_tol, int64_t* out_model);
/* NaiveBayesEstimator(numClasses, lambda).fit (K/nodes/learning/NaiveBayesModel.scala, MLlib's multinomial NaiveBayes.train):
 * W = theta^T with theta_cj = log(S_jc + lambda) - log(sum_j S_jc + d lambda), S_jc the sum of feature j over class c, and intercept
 * pi_c = log(n_c + lambda) - log(N + k lambda).  lambda finite and >= 0.  ks_last_fit_stats_json: solver "naive_bayes". */
KS_API int32_t ks_naive_bayes_fit(int64_t ctx, int64_t features_or_0, int64_t sparse_or_0, const int32_t* labels, int64_t n_labels,
                                  int32_t num_classes, double lambda, int64_t* out_model);

/* ---- the text front end (DESIGN.md section 23) ------------------------------------------------------------------------------------
 * Trim, LowerCase, Tokenizer, NGramsFeaturizer, TermFrequency, CommonSparseFeatures / AllSparseFeatures, SparseFeatureVectorizer,
 * HashingTF and NGramsHashingTF (K/nodes/nlp/StringUtils.scala, ngrams.scala, HashingTF.scala, NGramsHashingTF.scala,
 * K/nodes/stats/TermFrequency.scala, K/nodes/util/{Common,All}SparseFeatures.scala, SparseFeatureVectorizer.scala).  Text objects
 * (text, token and term-frequency batches, fitted feature spaces) share one handle space, released by ks_text_destroy; a text object
 * keeps the objects it was made from alive.  Orders: (0, 0) takes every token as a term of its own (a Java String); 1 <= min <= max
 * takes the n-grams of those orders (Scala Seqs of Strings), emitted per position i, then order.  Nothing here is collective. */
#define KS_TEXT_TRIM 1   /* Java String.trim: strip leading and trailing code points <= U+0020 */
#define KS_TEXT_LOWER 2  /* the one-to-one Unicode lowercase mapping per code point, U+0130 to U+0069 U+0307, no final-sigma rule */
/* ks_ctx_set_option "debug_text_hash_bits" (1..64, for tests): the content hashes keep only their low bits, forcing collisions.  It
 * is rejected once the context holds a text object, so that every object is hashed, sorted and looked up under one mask. */
/* A batch of n_docs documents: bytes (n_bytes of UTF-8) and doc_offsets (n_docs + 1, from 0 to n_bytes, non-decreasing).  Invalid
 * UTF-8 (a bad lead or continuation byte, an overlong form, a surrogate, a code point above U+10FFFF or a sequence that crosses a
 * document boundary) is found on the device and rejected with KS_ERR_INVALID. */
KS_API int32_t ks_text_from_host(int64_t ctx, const uint8_t* bytes, int64_t n_bytes, const int64_t* doc_offsets, int64_t n_docs,
                                 int64_t* out_text);
KS_API int32_t ks_text_transform(int64_t ctx, int64_t text, int32_t flags, int64_t* out_text);
/* Tokenizer() (Java String.split on [\p{Punct}\s]+): a leading separator gives a leading "", trailing empty tokens are dropped, an
 * empty document gives [""] and a document of separators only gives no token.  Per token the device also keeps Java's
 * String.hashCode (over UTF-16 code units) and a 64-bit content hash. */
KS_API int32_t ks_text_tokenize(int64_t ctx, int64_t text, int64_t* out_tokens);
/* A token batch from the host: token t is bytes[token_offsets[t], token_offsets[t + 1]); document d holds tokens
 * [doc_offsets[d], doc_offsets[d + 1]). */
KS_API int32_t ks_tokens_from_host(int64_t ctx, const uint8_t* bytes, int64_t n_bytes, const int64_t* token_offsets, int64_t n_tokens,
                                   const int64_t* doc_offsets, int64_t n_docs, int64_t* out_tokens);
/* TermFrequency over the terms of a token batch (orders as above, max_order <= 4): per document its distinct terms in order of first
 * occurrence, each with its count as value; *out_max_count is the largest count (0 without terms). */
KS_API int32_t ks_term_frequency(int64_t ctx, int64_t tokens, int32_t min_order, int32_t max_order, int64_t* out_tf,
                                 int64_t* out_max_count);
/* value = table[count - 1] for every term (n >= the largest count, every entry finite) */
KS_API int32_t ks_tf_set_weights(int64_t ctx, int64_t tf, const double* table, int64_t n);
/* A term-frequency batch from the host over the tokens of a token batch: term e is tokens [term_first[e], term_first[e] + max(order, 1))
 * of it, a String when term_order[e] is 0 and a Seq of term_order[e] <= 4 Strings otherwise, with value values[e] (finite);
 * document d holds terms [doc_offsets[d], doc_offsets[d + 1]). */
KS_API int32_t ks_tf_from_host(int64_t ctx, int64_t tokens, const int64_t* term_first, const int32_t* term_order, const double* values,
                               int64_t n_terms, const int64_t* doc_offsets, int64_t n_docs, int64_t* out_tf);
/* CommonSparseFeatures(num_features).fit, or AllSparseFeatures().fit with num_features = -1: the distinct terms ranked by the number of
 * entries that hold them (document frequency), descending, then by their first entry; the first num_features of them.  Terms are the
 * same feature exactly when their bytes are equal.  The space owns a copy of its terms.  KS_ERR_INVALID on a context with several
 * ranks (an exact top-K over ranks is not implemented) and for a batch without terms (a space has at least one feature). */
KS_API int32_t ks_sparse_features_fit(int64_t ctx, int64_t tf, int64_t num_features, int64_t* out_space);
/* A feature space from the host: feature f (column f) is the term (term_first[f], term_order[f]) over the tokens of a token batch. */
KS_API int32_t ks_sparse_features_from_host(int64_t ctx, int64_t tokens, const int64_t* term_first, const int32_t* term_order,
                                            int64_t n_features, int64_t* out_space);
/* SparseFeatureVectorizer.apply: a sparse matrix handle with one row per document and one column per feature, the value of every term
 * found in the space by its bytes (others dropped), columns ascending and distinct within a row: a term an uploaded batch repeats
 * within one document gives one entry, the sum of its values in entry order. */
KS_API int32_t ks_sparse_features_apply(int64_t ctx, int64_t space, int64_t tf, int64_t* out_sparse);
/* HashingTF(num_features) over the terms of a token batch (orders as above; no limit on max_order), which is NGramsHashingTF(orders,
 * num_features) for orders >= 1: a sparse matrix handle of counts at column nonNegativeMod(term.##, num_features), String.hashCode for
 * a String and MurmurHash3.seqHash for a Seq.  num_features in [1, INT32_MAX]. */
KS_API int32_t ks_hashing_tf(int64_t ctx, int64_t tokens, int32_t min_order, int32_t max_order, int64_t num_features, int64_t* out_sparse);
/* Host copies of a text object's arrays, for inspection.  KS_TEXT_BYTES (uint8): the UTF-8 the object's documents or tokens point
 * into; KS_TEXT_DOC_OFFSETS (int64, documents + 1): byte offsets of a text batch, token offsets of a token batch, term offsets of a
 * term-frequency batch; KS_TEXT_TOKEN_BEGIN / _END (int64): byte ranges of the tokens; KS_TEXT_TOKEN_JAVA_HASH (int32); KS_TEXT_TERM_FIRST
 * (int64), _ORDER (int32), _COUNT (int32), _VALUE (double): the terms of a term-frequency batch or the features of a space.
 * ks_text_array_size gives the element count (KS_ERR_INVALID: the object has no such array); ks_text_array copies n of them. */
#define KS_TEXT_BYTES 0
#define KS_TEXT_DOC_OFFSETS 1
#define KS_TEXT_TOKEN_BEGIN 2
#define KS_TEXT_TOKEN_END 3
#define KS_TEXT_TOKEN_JAVA_HASH 4
#define KS_TEXT_TERM_FIRST 5
#define KS_TEXT_TERM_ORDER 6
#define KS_TEXT_TERM_COUNT 7
#define KS_TEXT_TERM_VALUE 8
KS_API int32_t ks_text_array_size(int64_t ctx, int64_t obj, int32_t which, int64_t* out_n);
KS_API int32_t ks_text_array(int64_t ctx, int64_t obj, int32_t which, void* out, int64_t n);
KS_API int32_t ks_text_destroy(int64_t ctx, int64_t obj);


/* ---- covariance-based transforms (DESIGN.md section 15) -------------------------------------
 * Every product of these fits runs in fp64 on the DMMA tensor core; they take no precision mode.  The fitted objects are ordinary
 * model handles (apply, save / load, host views): apply runs in the context's precision like every model.  x: this rank's rows
 * (any rank may hold fewer than d rows, or none).  Rank 0's eigen / SVD / CholeskyQR factors are broadcast, so the models are
 * bit-identical across ranks.  All are collective. */
/* PCAEstimator(dims) / DistributedPCAEstimator(dims).fit (K/nodes/learning/PCA.scala:157-199, DistributedPCA.scala:30-56): eigenvectors
 * of the exactly centred covariance, descending, MATLAB sign convention, the first dims -> model (d x dims, no mean, no intercept:
 * PCATransformer does not centre).  dims in [1, d]. */
KS_API int32_t ks_pca_fit(int64_t ctx, int64_t x, int32_t dims, int64_t* out_model);
/* ZCAWhitenerEstimator(eps).fitSingle (K/nodes/learning/ZCAWhitener.scala:37-72) -> model (d x d whitener V diag(w) V^T with
 * w = (lambda / (N - 1) + eps)^-1/2, feature means = column means).  Needs N >= d rows over all ranks; eps finite and >= 0. */
KS_API int32_t ks_zca_fit(int64_t ctx, int64_t x, double eps, int64_t* out_model);
/* ApproximatePCAEstimator.approximateQ (K/nodes/learning/ApproximatePCA.scala:69-85): this rank's rows of the orthonormal N x l
 * basis, as an fp32 matrix.  omega: the caller's d x l Gaussian test matrix (column-major); l in [1, min(N, d)], q >= 0.  The QR of
 * every tall-skinny factor is shifted CholeskyQR3. */
KS_API int32_t ks_approx_range(int64_t ctx, int64_t x, const double* omega_colmajor /* d x l */, int32_t l, int32_t q, int64_t* out_q);
/* ApproximatePCAEstimator(dims, q, p).fit (ApproximatePCA.scala:37-58) with the caller's omega (d x (dims + p), column-major) ->
 * model (d x dims, no mean, no intercept).  No centring, like the reference. */
KS_API int32_t ks_approx_pca_fit(int64_t ctx, int64_t x, const double* omega_colmajor, int32_t dims, int32_t q, int32_t p,
                                 int64_t* out_model);

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
/* out (m x n, row-major fp64, ld_out) = (A - 1 s^T)^T (B - 1 t^T) through the fp64 DMMA Gram of the PCA fits; b = 0: symmetric mode
 * (B = A, t = s); either shift may be NULL (zero).  Not collective. */
KS_API int32_t ks_debug_gram_f64(int64_t ctx, int64_t a, int64_t b_or_0, const double* shift_a_or_null, const double* shift_b_or_null,
                                 double* out, int64_t ld_out);
/* The projection GEMM of generated features alone: feature columns [c0, c0 + cols) of rows [row_begin, row_begin + rows) of
 * x_in + rfs[n_rfs] (cosine or PaddedFFT maps), minus shift_or_null (cols values; NULL: zero), produced by the same feature
 * source and launch as in the fits.  The slab kinds are those the fits request:
 *   KS_PRECISION_TF32   tf32 operands, fp32 slab, tf32-rounded (round_out = 1) or unrounded (round_out = 0);
 *   KS_PRECISION_F16    fp16 slab of the __cosf value (round_out = 1, the blocks of the fits) or of the range-reduced cosine
 *                       (round_out = 0, their feature-mean estimates); fp16 operands, or tf32 operands when the option proj_f16 is 0;
 *   KS_PRECISION_F16X2  split operands, round_out = 0: the unrounded fp32 slab, or with out_lo the fp16 pair (hi -> out, lo -> out_lo).
 * Any other combination: KS_ERR_INVALID.  out / out_lo: rows x cols, row-major fp64 (ld_out); colsum_or_null (cols): the column
 * sums the kernel accumulates for the fits' feature means. */
KS_API int32_t ks_debug_slab(int64_t ctx, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int32_t precision, int32_t round_out,
                             int64_t row_begin, int64_t rows, int64_t c0, int64_t cols, const double* shift_or_null, double* out,
                             double* out_lo_or_null, int64_t ld_out, double* colsum_or_null);
/* Times `iters` launches of the projection alone (CUDA events; returns ms per launch): feature columns [0, cols) of all rows of
 * x_in + rfs[n_rfs], the slab kind as in ks_debug_slab (shift zero), launched as a block fit's first sweep launches it (on the
 * look-ahead stream, column sums on; for the fp16 pair also the exact Gram diagonal).  diag_or_null (KS_PRECISION_F16X2 only,
 * cols values): the fp64 sum of (hi + lo)^2 per column accumulated by the last launch.  out_or_null / out_lo_or_null (rows x cols,
 * row-major fp64): the slab of the last launch (the lo plane for KS_PRECISION_F16X2 only).  The option reserve_sms sets how many
 * SMs the launch leaves free, as in the fits. */
KS_API int32_t ks_debug_time_slab(int64_t ctx, int64_t x_in, const int64_t* rfs, int32_t n_rfs, int32_t precision, int32_t round_out,
                                  int64_t cols, int32_t iters, double* out_ms, double* diag_or_null, double* out_or_null,
                                  double* out_lo_or_null);
/* The residual-update / model-apply GEMM alone, launched as the fits launch it: out (M x N device matrix, updated in place)
 * = [out +] bias + sign * acc_scale * A B^T with A (M x K), B (N x K) device matrices; apply = 0: residual update (sign -1),
 * 1: model apply (sign +1); reduce = 1 adds into out, 0 overwrites it; bias_or_null: N values (NULL: zero); acc_scale: a power
 * of two, read by the kernel from device memory.  precision: KS_PRECISION_TF32 (fp32 operands as they are), KS_PRECISION_F16
 * (fp16 copies) or KS_PRECISION_F16X2 (fp16 pairs hi + lo, residual update only). */
KS_API int32_t ks_debug_update(int64_t ctx, int64_t a, int64_t b, int32_t apply, int32_t precision, const double* bias_or_null,
                               int32_t reduce, double acc_scale, int64_t out);
/* Arms the context: the next ks_blockwls_fit copies the fp64 system it assembles for class cls in feature block `block` during
 * the first sweep, before the Cholesky factorisation overwrites it: H (b x b, column-major, b = that block's width) into
 * H_out and the right-hand side (b) into rhs_out (either may be NULL, not both).  The host buffers must stay valid until
 * that fit returns; the fit disarms the context whether or not the class and block exist. */
KS_API int32_t ks_debug_bwls_capture(int64_t ctx, int32_t block, int32_t cls, double* H_out, double* rhs_out);
/* Adds step (sweep, block) to the steps the next ks_blockls_fit / ks_linear_map_fit on the context copies to the host; several
 * calls request several steps of one fit.  outs[KS_BLS_CAP_COUNT]: host buffers indexed by the KS_BLS_CAP_* constants, each
 * NULL (not wanted) or large enough for its entry below, with b that block's width, n the context's row count, k the classes.
 * Every entry is fp64, converted exactly from what the device holds, and copied on the stream that produced it at the point
 * listed, so the fit launches the same kernels with and without a capture.  The buffers must stay valid until that fit
 * returns; the fit disarms the context whether or not the steps exist.  H and DIAG exist at sweep 0 only (later sweeps reuse
 * the cached factor): requesting them for a later sweep is KS_ERR_INVALID.  The copies block the host between collectives, so
 * with several ranks arm the same steps on every rank. */
#define KS_BLS_CAP_SHIFT 0     /* b: the fp32 shift m_j the slab was built with, after the shift estimate */
#define KS_BLS_CAP_DELTA 1     /* b: delta_j = mean(slab) as launch_delta_mean wrote it (mean_j = m_j + delta_j), copied in the
                                  solve chain with RHS, after it has waited for the factor */
#define KS_BLS_CAP_DIAG 2      /* b: the exact fp64 diagonal of S^T S, all-reduced (parity mode only), before the system assembly */
#define KS_BLS_CAP_H 3         /* b x b column-major: H_j = S^T S - N delta delta^T + lambda I before the Cholesky factorisation */
#define KS_BLS_CAP_RHS 4       /* b x k column-major: S^T R - delta rsum^T - lambda W_old, before the solve */
#define KS_BLS_CAP_DW 5        /* b x k column-major: the increment dW_j, after the solve, before it is packed for the update */
#define KS_BLS_CAP_SLAB_HI 6   /* n x b row-major: the slab S_j (hi plane of the split operands) as the Gram kernels read it */
#define KS_BLS_CAP_SLAB_LO 7   /* n x b row-major: its lo plane (zero in the single-operand modes) */
#define KS_BLS_CAP_R_BEFORE 8  /* n x k row-major: the fp32 residual before this step's C = S^T R */
#define KS_BLS_CAP_R_AFTER 9   /* n x k row-major: the fp32 residual after this step's update R -= (S - 1 delta^T) dW */
#define KS_BLS_CAP_SCALES 10   /* 4: fp16 modes' powers of two {residual s, 1/s, increment s, 1/s} (1 otherwise), with DW */
#define KS_BLS_CAP_COUNT 11
KS_API int32_t ks_debug_blockls_capture(int64_t ctx, int32_t sweep, int32_t block, double* const* outs);

/* X = H^-1 B for a symmetric positive definite H (column-major n x n) and B (column-major n x k): Cholesky with cuSOLVER, then
 * either the library's own multi-RHS solve kernel (use_cusolver = 0; option "custom_solve") or cusolverDnDpotrs (the default of
 * the fits); best-of-3 ms. */
KS_API int32_t ks_debug_chol_solve(int64_t ctx, const double* H_colmajor, int32_t n, const double* B_colmajor, int32_t k,
                                   int32_t use_cusolver, double* X_out, double* out_ms);

#ifdef __cplusplus
}
#endif
#endif /* KEYSTONE_B200_H */
