package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.GaussianMixtureModel
import keystoneml.workflow.Transformer
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.images.FisherVector(gmm) followed by MatrixVectorizer: one vectorised D x 2K Fisher vector per
 * (D x n_i) descriptor matrix, posteriors and statistics in fp64 on this executor's GPU (DESIGN.md section 16; fv2 follows Sanchez
 * et al., not the transposed term of FisherVector.scala:47).  The RDD apply encodes each partition's items in one device call.
 * Not collective.  Not compiled in the build image (no JVM).
 */
class GpuFisherVector(val gmm: GaussianMixtureModel, job: GpuJob) extends Transformer[DenseMatrix[Float], DenseVector[Float]] {

  /** One device call for a batch of items; returns one vector of 2 D K values per item (element (d, j) at d + D j). */
  def applyBatch(items: Array[DenseMatrix[Float]]): Array[DenseVector[Float]] = {
    val lib = GpuExecutor.lib
    val c = GpuExecutor.ctx(job.deviceOf(0), 0, 1, null)
    val (d, k) = (gmm.means.rows, gmm.means.cols)
    val offs = items.scanLeft(0L)((o, m) => o + m.cols)
    val rows = offs.last
    val x = lib.matrixCreate(c, rows, d)
    items.zip(offs).foreach { case (m, o) =>   // item columns become device rows: DenseMatrix.data of the D x n item, row-major n x D
      if (m.cols > 0) lib.matrixWriteRows(c, x, o, convert(m, Double).toDenseMatrix.copy.data, m.cols, d)
    }
    val g = lib.gmmCreate(c, gmm.means.copy.data, gmm.variances.copy.data, gmm.weights.toArray, d, k, gmm.weightThreshold)
    val fv = lib.fisherVectorApply(c, g, x, offs)
    val host = lib.matrixToHost(c, fv)
    lib.matrixDestroy(c, fv); lib.gmmDestroy(c, g); lib.matrixDestroy(c, x)
    val per = 2 * d * k
    items.indices.map(i => DenseVector(host.slice(i * per, (i + 1) * per).map(_.toFloat))).toArray
  }

  override def apply(in: DenseMatrix[Float]): DenseVector[Float] = applyBatch(Array(in))(0)

  override def apply(in: RDD[DenseMatrix[Float]]): RDD[DenseVector[Float]] = in.mapPartitions { it =>
    val items = it.toArray
    if (items.isEmpty) Iterator.empty else applyBatch(items).iterator
  }
}
