package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.KMeansModel
import keystoneml.utils.MatrixUtils
import keystoneml.workflow.Estimator
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.learning.KMeansPlusPlusEstimator: k-means++ seeding and Lloyd passes in fp64 on this executor's GPU
 * (DESIGN.md section 17).  Returns the reference's own KMeansModel (numMeans x dim means).  The seeding uniforms come from
 * java.util.Random(seed); the reference's MersenneTwister / Multinomial stream is not reproduced.  Not compiled in the build image
 * (no JVM).
 */
case class GpuKMeansPlusPlusEstimator(numMeans: Int, maxIterations: Int, job: GpuJob, stopTolerance: Double = 1e-3, seed: Int = 0)
  extends Estimator[DenseVector[Double], DenseVector[Double]] {

  def fit(data: RDD[DenseVector[Double]]): KMeansModel = fit(MatrixUtils.rowsToMatrix(data.collect()))

  def fit(X: DenseMatrix[Double]): KMeansModel = {
    val lib = GpuExecutor.lib
    val c = GpuExecutor.ctx(job.deviceOf(0), 0, 1, null)
    val x = lib.matrixCreate(c, X.rows, X.cols)
    lib.matrixWriteRows(c, x, 0, X.t.copy.data, X.rows, X.cols)  // row-major rows x cols
    val rand = new java.util.Random(seed)
    val means = new Array[Double](numMeans * X.cols)
    lib.kmeansFit(c, x, numMeans, maxIterations, stopTolerance, Array.fill(numMeans)(rand.nextDouble()), means)
    lib.matrixDestroy(c, x)
    KMeansModel(new DenseMatrix(X.cols, numMeans, means).t.copy)  // row-major numMeans x dim
  }
}
