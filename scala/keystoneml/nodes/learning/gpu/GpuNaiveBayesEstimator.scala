package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.NaiveBayesModel
import keystoneml.workflow.LabelEstimator
import org.apache.spark.rdd.RDD

import scala.reflect.ClassTag

/**
 * Drop-in for keystoneml.nodes.learning.NaiveBayesEstimator (NaiveBayesModel.scala): the reference's constructor arguments followed
 * by the GPU job, the same fit signature and the same returned NaiveBayesModel(labels, pi, theta).  The fit is the collective
 * ks_naive_bayes_fit (MLlib's multinomial formulas, DESIGN.md section 22); a class with no rows is an error rather than a smaller
 * model.  Not compiled in the build image (no JVM).
 */
case class GpuNaiveBayesEstimator[T <: Vector[Double] : ClassTag](numClasses: Int, lambda: Double = 1.0, job: GpuJob)
    extends LabelEstimator[T, DenseVector[Double], Int] {

  override def fit(in: RDD[T], labels: RDD[Int]): NaiveBayesModel[T] = {
    val (k, lam) = (numClasses, lambda)
    val (w, pi) = GpuClassifierFit(in, labels, job, (lib, c, f, s, y) => lib.naiveBayesFit(c, f, s, y, k, lam))
    val theta = Array.tabulate(k)(c => w(::, c).toArray)
    new NaiveBayesModel[T]((0 until k).toArray, pi, theta)
  }
}
