package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.LogisticRegressionModel
import keystoneml.workflow.LabelEstimator
import org.apache.spark.mllib.classification.{LogisticRegressionModel => MLlibLRM}
import org.apache.spark.mllib.linalg.Vectors
import org.apache.spark.rdd.RDD

import scala.reflect.ClassTag

/**
 * Drop-in for keystoneml.nodes.learning.LogisticRegressionEstimator (LogisticRegressionModel.scala): the reference's constructor
 * arguments in its order, followed by the GPU job; the same fit signature and the same returned LogisticRegressionModel wrapping an
 * MLlib model (weights class-major, (k - 1) * d; intercept 0).  The fit is the collective ks_logistic_fit: MLlib's LogisticGradient
 * with SquaredL2Updater, no intercept, by L-BFGS with a strong-Wolfe line search in fp64 (DESIGN.md section 22).  convergenceTol is
 * honoured.  Not compiled in the build image (no JVM).
 */
case class GpuLogisticRegressionEstimator[T <: Vector[Double] : ClassTag](numClasses: Int, regParam: Double = 0, numIters: Int = 100,
    convergenceTol: Double = 1E-4, numFeatures: Int = -1, job: GpuJob) extends LabelEstimator[T, Double, Int] {

  require(numClasses > 1)

  override def fit(in: RDD[T], labels: RDD[Int]): LogisticRegressionModel[T] = {
    val (k, lam, it, tol) = (numClasses, regParam, numIters, convergenceTol)
    val (w, _) = GpuClassifierFit(in, labels, job, (lib, c, f, s, y) => lib.logisticFit(c, f, s, y, k, lam, it, tol))
    require(numFeatures == -1 || numFeatures == w.rows, s"numFeatures is $numFeatures but the data has ${w.rows} features")
    val weights = w(::, 1 until k).t.copy.toDenseVector   // column 0 is the pivot class; class-major like MLlib's weights
    val model = if (k == 2) new MLlibLRM(Vectors.dense(weights.toArray), 0.0)
    else new MLlibLRM(Vectors.dense(weights.toArray), 0.0, w.rows, k)
    new LogisticRegressionModel[T](model)
  }
}
