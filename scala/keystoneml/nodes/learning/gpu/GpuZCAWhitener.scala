package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.ZCAWhitener
import keystoneml.workflow.Estimator
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.learning.ZCAWhitenerEstimator (ZCAWhitener.scala:30-72): fitSingle uploads the sample matrix to one
 * GPU (a one-rank context) and returns the reference's ZCAWhitener(whitener, means); fit uses the first item, like the reference.
 * The covariance, its eigenpairs and the whitener are fp64 on the device (DESIGN.md section 15).  Needs at least d rows.
 * Not compiled in the build image (no JVM).
 */
class GpuZCAWhitenerEstimator(val eps: Double = 0.1, job: GpuJob) extends Estimator[DenseMatrix[Double], DenseMatrix[Double]] {

  def fit(in: RDD[DenseMatrix[Double]]): ZCAWhitener = fitSingle(in.first)

  def fitSingle(in: DenseMatrix[Double]): ZCAWhitener = {
    val lib = GpuExecutor.lib
    val c = GpuExecutor.ctx(job.deviceOf(0), 0, 1, null)
    val d = in.cols
    val x = lib.matrixCreate(c, in.rows, d)
    lib.matrixWriteRows(c, x, 0, in.t.copy.data, in.rows, d)   // row-major
    val h = lib.zcaFit(c, x, eps)
    val nb = lib.modelNumBlocks(c, h)
    val w = DenseMatrix.vertcat((0 until nb).map(j => lib.modelGetBlock(c, h, j)).map(b => new DenseMatrix[Double](b.length / d, d, b)): _*)
    val means = DenseVector((0 until nb).flatMap(j => lib.modelGetBlockMean(c, h, j)).toArray)
    lib.modelDestroy(c, h); lib.matrixDestroy(c, x)
    new ZCAWhitener(w, means)
  }
}
