package keystoneml.nodes.learning.gpu

/**
 * JNI binding of libkeystone_b200 (include/keystone_b200.h via jni/keystone_b200_jni.cpp).
 * Same convention as the reference's only native nodes (keystoneml.utils.external.VLFeat / EncEval):
 * a Serializable class whose constructor loads the library, @native methods on primitives and primitive arrays.
 * Every failed call throws a RuntimeException carrying ks_last_error().
 * Not compiled in the build image (no JVM); kept mechanical so it can be checked against the C header by eye.
 */
class KeystoneB200 extends Serializable {
  System.loadLibrary("keystone_b200_jni") // run-pipeline.sh passes -Djava.library.path=$FWDIR/lib

  @native def ncclUniqueId(): Array[Byte]
  @native def ctxCreate(device: Int, rank: Int, world: Int, ncclId: Array[Byte]): Long
  @native def ctxDestroy(ctx: Long): Unit
  @native def ctxSetOption(ctx: Long, name: String, value: Long): Unit

  @native def matrixCreate(ctx: Long, nRows: Long, nCols: Long): Long
  @native def matrixWriteRows(ctx: Long, m: Long, row0: Long, rowMajor: Array[Double], nRows: Long, nCols: Long): Unit
  @native def labelsFromClasses(ctx: Long, classes: Array[Int], numClasses: Int): Long
  @native def matrixToHost(ctx: Long, m: Long): Array[Double]
  @native def matrixDestroy(ctx: Long, m: Long): Unit

  @native def cosineRfCreate(ctx: Long, w: Array[Double], b: Array[Double], nOut: Long, nIn: Long): Long
  @native def paddedFftCreate(ctx: Long, signs: Array[Double], nIn: Long, rectify: Boolean, maxVal: Double, alpha: Double): Long
  @native def featureMapApply(ctx: Long, rf: Long, xIn: Long): Long
  @native def featureMapDestroy(ctx: Long, rf: Long): Unit

  /** precisionMode: KeystoneB200.PrecisionDefault (-1: the context's, initially the parity mode), 0 tf32, 1 fp16, 2 split operands. */
  @native def blockLsFit(ctx: Long, features: Long, xIn: Long, rfs: Array[Long], labels: Long,
      blockSize: Int, numIter: Int, lambda: Double, numFeaturesOr0: Long, precisionMode: Int): Long
  @native def blockWlsFit(ctx: Long, features: Long, xIn: Long, rfs: Array[Long], labels: Long,
      blockSize: Int, numIter: Int, lambda: Double, mixtureWeight: Double, numFeaturesOr0: Long, precisionMode: Int): Long
  @native def linearMapFit(ctx: Long, features: Long, labels: Long, hasLambda: Boolean, lambda: Double): Long
  @native def lbfgsFit(ctx: Long, features: Long, xIn: Long, rfs: Array[Long], labels: Long, fitIntercept: Boolean,
      numCorrections: Int, convergenceTol: Double, numIterations: Int, regParam: Double, precisionMode: Int): Long
  /** Sparse rows as CSR (indptr: nRows + 1 offsets; indices / values: indptr(nRows) each), their Densify, SparseLBFGSwithL2 and
   *  SparseLinearMapper.apply (DESIGN.md section 20).  A sparse handle is not a matrix handle. */
  @native def sparseFromHostCsr(ctx: Long, indptr: Array[Long], indices: Array[Int], values: Array[Double], nCols: Long): Long
  @native def sparseDestroy(ctx: Long, s: Long): Unit
  @native def sparseDensify(ctx: Long, s: Long): Long
  @native def sparseLbfgsFit(ctx: Long, s: Long, labels: Long, fitIntercept: Boolean, numCorrections: Int, convergenceTol: Double,
      numIterations: Int, regParam: Double): Long
  @native def modelApplySparse(ctx: Long, model: Long, s: Long): Long
  /** LogisticRegressionEstimator / NaiveBayesEstimator (collective): exactly one of features and sparse is a handle, the other 0. */
  @native def logisticFit(ctx: Long, features: Long, sparse: Long, classes: Array[Int], numClasses: Int, regParam: Double, numIters: Int,
      convergenceTol: Double): Long
  @native def naiveBayesFit(ctx: Long, features: Long, sparse: Long, classes: Array[Int], numClasses: Int, lambda: Double): Long
  /** The text front end (DESIGN.md section 23; not collective): UTF-8 bytes with Long offsets in, text-object handles out (released
   *  by textDestroy).  termFrequency returns (handle, largest count); textArray* read a KS_TEXT_* array of an object back;
   *  sparseFeaturesApply and hashingTf return sparse matrix handles, read by sparseToHostCsr as (indptr, indices, values). */
  @native def textFromHost(ctx: Long, bytes: Array[Byte], docOffsets: Array[Long]): Long
  @native def textTransform(ctx: Long, text: Long, flags: Int): Long
  @native def textTokenize(ctx: Long, text: Long): Long
  @native def tokensFromHost(ctx: Long, bytes: Array[Byte], tokenOffsets: Array[Long], docOffsets: Array[Long]): Long
  @native def termFrequency(ctx: Long, tokens: Long, minOrder: Int, maxOrder: Int): Array[Long]
  @native def tfSetWeights(ctx: Long, tf: Long, table: Array[Double]): Unit
  @native def tfFromHost(ctx: Long, tokens: Long, termFirst: Array[Long], termOrder: Array[Int], values: Array[Double],
      docOffsets: Array[Long]): Long
  @native def sparseFeaturesFit(ctx: Long, tf: Long, numFeatures: Long): Long
  @native def sparseFeaturesFromHost(ctx: Long, tokens: Long, termFirst: Array[Long], termOrder: Array[Int]): Long
  @native def sparseFeaturesApply(ctx: Long, space: Long, tf: Long): Long
  @native def hashingTf(ctx: Long, tokens: Long, minOrder: Int, maxOrder: Int, numFeatures: Long): Long
  @native def textArrayBytes(ctx: Long, obj: Long, which: Int): Array[Byte]
  @native def textArrayInts(ctx: Long, obj: Long, which: Int): Array[Int]
  @native def textArrayLongs(ctx: Long, obj: Long, which: Int): Array[Long]
  @native def textArrayDoubles(ctx: Long, obj: Long, which: Int): Array[Double]
  @native def textDestroy(ctx: Long, obj: Long): Unit
  @native def sparseToHostCsr(ctx: Long, s: Long): Array[AnyRef]
  /** PCA / ZCA / approximate PCA (collective, fp64 on the device); omega is the d x l test matrix, DenseMatrix.data. */
  @native def pcaFit(ctx: Long, x: Long, dims: Int): Long
  @native def zcaFit(ctx: Long, x: Long, eps: Double): Long
  @native def approxRange(ctx: Long, x: Long, omega: Array[Double], l: Int, q: Int): Long
  @native def approxPcaFit(ctx: Long, x: Long, omega: Array[Double], dims: Int, q: Int, p: Int): Long
  /** LCS descriptors, GMM posteriors, Fisher vectors (not collective; DESIGN.md section 16).  means / variances: D x K
   *  DenseMatrix.data; itemOffsets: nItems + 1 row offsets into the descriptor matrix. */
  @native def lcsExtract(ctx: Long, images: Long, xDim: Int, yDim: Int, channels: Int, stride: Int, strideStart: Int,
      subPatchSize: Int): Long
  @native def gmmCreate(ctx: Long, means: Array[Double], variances: Array[Double], weights: Array[Double], dim: Long, k: Long,
      weightThreshold: Double): Long
  @native def gmmDestroy(ctx: Long, gmm: Long): Unit
  @native def gmmPosteriors(ctx: Long, gmm: Long, x: Long): Long
  @native def fisherVectorApply(ctx: Long, gmm: Long, descriptors: Long, itemOffsets: Array[Long]): Long
  @native def matrixNormalizeRows(ctx: Long, m: Long): Long
  /** GMM EM, k-means++ and the row gather (not collective; DESIGN.md section 17).  uniforms: the header's draw rule; GMM means /
   *  variances out: D x K DenseMatrix.data; k-means means out: numMeans x dim row-major. */
  @native def gmmFit(ctx: Long, x: Long, k: Long, maxIterations: Int, minClusterSize: Double, stopTolerance: Double,
      weightThreshold: Double, smallVarianceThreshold: Double, absoluteVarianceThreshold: Double, initialization: Int,
      uniforms: Array[Double], meansOut: Array[Double], variancesOut: Array[Double], weightsOut: Array[Double]): Long
  @native def kmeansFit(ctx: Long, x: Long, numMeans: Long, maxIterations: Int, stopTolerance: Double, uniforms: Array[Double],
      meansOut: Array[Double]): Int
  @native def kmeansAssign(ctx: Long, x: Long, meansRowMajor: Array[Double], numMeans: Long, dim: Long): Long
  @native def matrixGatherRows(ctx: Long, m: Long, rows: Array[Long]): Long
  @native def matrixSignedSqrt(ctx: Long, m: Long): Long
  /** PixelScaler, GrayScaler and dense SIFT (not collective; DESIGN.md section 18).  siftKeypoints is host only: the per-scale
   *  keypoint counts, or null for rejected arguments. */
  @native def imagePixelScale(ctx: Long, images: Long): Long
  @native def imageGrayscale(ctx: Long, images: Long, xDim: Int, yDim: Int, channels: Int, pixelScale: Int): Long
  @native def siftExtract(ctx: Long, grayImages: Long, xDim: Int, yDim: Int, step: Int, bin: Int, scales: Int, scaleStep: Int): Long
  @native def siftKeypoints(xDim: Int, yDim: Int, step: Int, bin: Int, scales: Int, scaleStep: Int): Array[Long]
  /** HOG (pixelScale = 1 takes PixelScaler's x / 255.0 in fp64) and DAISY (not collective; DESIGN.md section 19). */
  @native def hogExtract(ctx: Long, images: Long, xDim: Int, yDim: Int, channels: Int, pixelScale: Int, bin: Int): Long
  @native def daisyExtract(ctx: Long, grayImages: Long, xDim: Int, yDim: Int, daisyT: Int, daisyQ: Int, daisyR: Int, daisyH: Int,
      pixelBorder: Int, stride: Int): Long

  @native def modelFromHost(ctx: Long, xs: Array[Array[Double]], blockSize: Int, k: Long, b: Array[Double],
      means: Array[Array[Double]]): Long
  @native def modelNumBlocks(ctx: Long, model: Long): Int
  @native def modelGetBlock(ctx: Long, model: Long, j: Int): Array[Double]
  @native def modelGetBlockMean(ctx: Long, model: Long, j: Int): Array[Double]
  @native def modelGetIntercept(ctx: Long, model: Long): Array[Double]
  @native def modelApply(ctx: Long, model: Long, features: Long, xIn: Long, rfs: Array[Long]): Long
  @native def modelApplyArgmax(ctx: Long, model: Long, features: Long, xIn: Long, rfs: Array[Long], nRows: Long): Array[Int]
  @native def modelSave(ctx: Long, model: Long, path: String): Unit
  @native def modelLoad(ctx: Long, path: String): Long
  @native def modelDestroy(ctx: Long, model: Long): Unit

  // Gaussian-kernel ridge regression (KernelGenerator / KernelRidgeRegression / KernelBlockLinearMapper)
  @native def gaussianKernelCreate(ctx: Long, xTrain: Long, gamma: Double): Long
  @native def gaussianKernelBlock(ctx: Long, kernel: Long, x: Long, col0: Long, cols: Long): Long
  @native def gaussianKernelNumTrain(ctx: Long, kernel: Long): Long
  @native def gaussianKernelDestroy(ctx: Long, kernel: Long): Unit
  @native def krrFit(ctx: Long, kernel: Long, labels: Long, lambda: Double, blockSize: Int, numEpochs: Int,
                     blockOrder: Array[Int]): Long
  @native def kernelModelFromHost(ctx: Long, kernel: Long, xs: Array[Array[Double]], k: Long, blockSize: Int): Long
}

object KeystoneB200 {
  val PrecisionDefault = -1
  val PrecisionTf32 = 0
  val PrecisionF16 = 1
  val PrecisionSplit = 2
}
