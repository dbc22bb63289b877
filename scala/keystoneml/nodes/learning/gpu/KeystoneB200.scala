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
