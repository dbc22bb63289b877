package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.{GMMInitializationMethod, GaussianMixtureModel, KMEANS_PLUS_PLUS_INITIALIZATION}
import keystoneml.utils.MatrixUtils
import keystoneml.workflow.Estimator
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.learning.GaussianMixtureModelEstimator: diagonal-covariance EM in fp64 on this executor's GPU
 * (DESIGN.md section 17), started from k-means++ (one Lloyd pass) or from random means.  Returns the reference's own
 * GaussianMixtureModel (default weightThreshold 1e-4, as the reference's fit returns).  The uniforms come from
 * java.util.Random(seed); the reference's MersenneTwister / Multinomial stream is not reproduced.  Like the reference, the sample
 * is collected to the driver and fitted there.  Not compiled in the build image (no JVM).
 */
case class GpuGaussianMixtureModelEstimator(
    k: Int,
    job: GpuJob,
    maxIterations: Int = 100,
    minClusterSize: Int = 40,
    stopTolerance: Double = 1e-4,
    weightThreshold: Double = 1e-4,
    smallVarianceThreshold: Double = 1e-2,
    absoluteVarianceThreshold: Double = 1e-9,
    initializationMethod: GMMInitializationMethod = KMEANS_PLUS_PLUS_INITIALIZATION,
    seed: Int = 0)
  extends Estimator[DenseVector[Double], DenseVector[Double]] {
  require(minClusterSize > 0, "Minimum cluster size must be positive")
  require(maxIterations > 0, "maxIterations must be positive")

  def fit(samples: RDD[DenseVector[Double]]): GaussianMixtureModel = fit(samples.collect())

  def fit(samples: Array[DenseVector[Double]]): GaussianMixtureModel = {
    require(samples.length > 0, "Must have training points")
    val lib = GpuExecutor.lib
    val c = GpuExecutor.ctx(job.deviceOf(0), 0, 1, null)
    val d = samples(0).length
    val x = lib.matrixCreate(c, samples.length, d)
    lib.matrixWriteRows(c, x, 0, MatrixUtils.rowsToMatrix(samples).t.copy.data, samples.length, d)  // row-major n x d
    val rand = new java.util.Random(seed)
    val random = initializationMethod != KMEANS_PLUS_PLUS_INITIALIZATION
    val uniforms = Array.fill(if (random) k * d else k)(rand.nextDouble())
    val (means, vars, weights) = (new Array[Double](d * k), new Array[Double](d * k), new Array[Double](k))
    val g = lib.gmmFit(c, x, k, maxIterations, minClusterSize.toDouble, stopTolerance, weightThreshold, smallVarianceThreshold,
      absoluteVarianceThreshold, if (random) 1 else 0, uniforms, means, vars, weights)
    lib.gmmDestroy(c, g); lib.matrixDestroy(c, x)
    GaussianMixtureModel(new DenseMatrix(d, k, means), new DenseMatrix(d, k, vars), DenseVector(weights))
  }
}
