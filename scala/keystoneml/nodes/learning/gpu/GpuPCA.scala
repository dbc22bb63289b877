package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.PCATransformer
import keystoneml.workflow.Estimator
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.learning.PCAEstimator / DistributedPCAEstimator (PCA.scala:157-225, DistributedPCA.scala:20-74)
 * and ApproximatePCAEstimator (ApproximatePCA.scala:21-58): the same fit signature and the same PCATransformer(pcaMat), laid out
 * like GpuBlockLeastSquaresEstimator (one partition group per GPU, rows uploaded where they are, a barrier stage for the collective
 * fit, rank 0 returns the d x dims matrix).  The covariance (or the sketch products) run in fp64 on the device (DESIGN.md
 * section 15).  approximate = true runs ApproximatePCA with q, p and a Gaussian test matrix drawn from `seed` on the driver
 * (Breeze's MersenneTwister stream of the reference is not reproduced).
 * Not compiled in the build image (no JVM).
 */
class GpuPCAEstimator(dims: Int, job: GpuJob, approximate: Boolean = false, q: Int = 10, p: Int = 5, seed: Int = 0)
  extends Estimator[DenseVector[Float], DenseVector[Float]] {

  override def fit(samples: RDD[DenseVector[Float]]): PCATransformer = {
    val world = job.world
    val d = samples.first().length
    val omega: Array[Double] = if (approximate) {
      val rnd = new java.util.Random(seed)
      Array.fill(d * (dims + p))(rnd.nextGaussian())
    } else null
    val (k, jb, appr, qq, pp) = (dims, job, approximate, q, p)
    val mats = samples.coalesce(world).barrier().mapPartitions { rowsIt =>
      val tc = org.apache.spark.BarrierTaskContext.get()
      val rank = tc.partitionId()
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(rank), rank, jb.world, jb.ncclId)
      val rows = rowsIt.map(v => convert(v, Double)).toArray
      val x = lib.matrixCreate(c, rows.length, d)
      if (rows.nonEmpty) lib.matrixWriteRows(c, x, 0, GpuExecutor.flatten(rows), rows.length, d)
      tc.barrier()
      val h = if (appr) lib.approxPcaFit(c, x, omega, k, qq, pp) else lib.pcaFit(c, x, k)   // collective
      val out = if (rank == 0) Iterator.single((0 until lib.modelNumBlocks(c, h)).map(j => lib.modelGetBlock(c, h, j)).toArray)
        else Iterator.empty
      lib.modelDestroy(c, h); lib.matrixDestroy(c, x)
      out
    }.collect()
    val pca = DenseMatrix.vertcat(mats.head.map(w => new DenseMatrix[Double](w.length / dims, dims, w)): _*)  // feature blocks
    new PCATransformer(convert(pca, Float))
  }
}
