package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.{LeastSquaresDenseGradient, LinearMapper}
import keystoneml.nodes.learning.Gradient.DenseGradient
import keystoneml.nodes.stats.StandardScalerModel
import keystoneml.workflow.{LabelEstimator, WeightedNode}
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.learning.DenseLBFGSwithL2 (LBFGS.scala:135-192): the reference's constructor arguments in its
 * order, followed by the GPU job and the precision mode; the gradient must be a LeastSquaresDenseGradient, the only dense
 * gradient the reference has.  Same fit signature, same returned LinearMapper(W, Some(labelMean), Some(featureScaler)) or
 * LinearMapper(W, None, None).  The body replaces the StandardScaler passes and Breeze's L-BFGS by one
 * ks_lbfgs_fit call per executor, laid out exactly like GpuBlockLeastSquaresEstimator: one partition group per GPU, rows
 * uploaded where they are, a barrier stage for the collective fit, rank 0 returns the model arrays.  The steps are exact
 * minimisers along the L-BFGS directions instead of Breeze's line search (DESIGN.md section 14).
 * Not compiled in the build image (no JVM).
 */
class GpuDenseLBFGSwithL2(val gradient: DenseGradient, fitIntercept: Boolean = true, numCorrections: Int = 10,
    convergenceTol: Double = 1e-4, numIterations: Int = 100, regParam: Double = 0.0, job: GpuJob,
    precisionMode: Int = KeystoneB200.PrecisionDefault)
  extends LabelEstimator[DenseVector[Double], DenseVector[Double], DenseVector[Double]] with WeightedNode {

  require(gradient.isInstanceOf[LeastSquaresDenseGradient], "GpuDenseLBFGSwithL2 supports LeastSquaresDenseGradient only")

  override val weight = numIterations + 1

  override def fit(trainingFeatures: RDD[DenseVector[Double]], trainingLabels: RDD[DenseVector[Double]]): LinearMapper[DenseVector[Double]] = {
    val world = job.world
    val zipped = trainingFeatures.zip(trainingLabels).coalesce(world)
    val (fi, m, tol, it, lam, prec, jb) = (fitIntercept, numCorrections, convergenceTol, numIterations, regParam, precisionMode, job)
    val models = zipped.barrier().mapPartitions { rowsIt =>
      val tc = org.apache.spark.BarrierTaskContext.get()
      val rank = tc.partitionId()
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(rank), rank, jb.world, jb.ncclId)
      val rows = rowsIt.toArray
      val d = if (rows.isEmpty) 0 else rows(0)._1.length
      val k = if (rows.isEmpty) 0 else rows(0)._2.length
      val f = lib.matrixCreate(c, rows.length, d)
      val y = lib.matrixCreate(c, rows.length, k)
      val chunk = 65536
      var r0 = 0
      while (r0 < rows.length) {
        val r1 = math.min(rows.length, r0 + chunk)
        lib.matrixWriteRows(c, f, r0, GpuExecutor.flatten(rows.slice(r0, r1).map(_._1)), r1 - r0, d)
        lib.matrixWriteRows(c, y, r0, GpuExecutor.flatten(rows.slice(r0, r1).map(_._2)), r1 - r0, k)
        r0 = r1
      }
      tc.barrier()
      val h = lib.lbfgsFit(c, f, 0L, null, y, fi, m, tol, it, lam, prec)          // collective: NCCL all-reduce of A^T R inside
      val out = if (rank == 0) {
        val nb = lib.modelNumBlocks(c, h)
        Iterator.single((
          (0 until nb).map(j => lib.modelGetBlock(c, h, j)).toArray,
          if (fi) (0 until nb).map(j => lib.modelGetBlockMean(c, h, j)).toArray else Array.empty[Array[Double]],
          if (fi) lib.modelGetIntercept(c, h) else null, k))
      } else Iterator.empty
      lib.modelDestroy(c, h); lib.matrixDestroy(c, f); lib.matrixDestroy(c, y)
      out
    }.collect()
    val (ws, mus, b, k) = models.head
    val x = DenseMatrix.vertcat(ws.map(w => new DenseMatrix[Double](w.length / k, k, w)): _*)   // feature blocks, in order
    if (fitIntercept) {
      new LinearMapper[DenseVector[Double]](x, Some(DenseVector(b)), Some(new StandardScalerModel(DenseVector(mus.flatten), None)))
    } else {
      new LinearMapper[DenseVector[Double]](x, None, None)
    }
  }
}
