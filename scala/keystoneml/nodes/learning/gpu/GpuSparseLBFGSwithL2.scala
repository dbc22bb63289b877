package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.{LeastSquaresSparseGradient, SparseLinearMapper}
import keystoneml.nodes.learning.Gradient.SparseGradient
import keystoneml.workflow.{LabelEstimator, WeightedNode}
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.learning.SparseLBFGSwithL2 (LBFGS.scala:208-281): the reference's constructor arguments in its
 * order, followed by the GPU job; the gradient must be a LeastSquaresSparseGradient.  Same fit signature, same returned
 * SparseLinearMapper(W, Some(b)) or SparseLinearMapper(W, None).  Each executor packs its partition's SparseVectors into CSR arrays
 * (indptr, column indices, values; the active entries in storage order), uploads them with ks_sparse_from_host_csr, and a barrier
 * stage runs the collective ks_sparse_lbfgs_fit; rank 0 returns the model arrays.  The ones column of the intercept is implicit
 * and its bias is regularised like the weights; the steps are exact minimisers along the L-BFGS directions (DESIGN.md section 20).
 * Not compiled in the build image (no JVM).
 */
class GpuSparseLBFGSwithL2(val gradient: SparseGradient, fitIntercept: Boolean = true, numCorrections: Int = 10,
    convergenceTol: Double = 1e-4, numIterations: Int = 100, regParam: Double = 0.0, sparseOverhead: Double = 8, job: GpuJob)
  extends LabelEstimator[SparseVector[Double], DenseVector[Double], DenseVector[Double]] with WeightedNode {

  require(gradient.isInstanceOf[LeastSquaresSparseGradient], "GpuSparseLBFGSwithL2 supports LeastSquaresSparseGradient only")

  override val weight = numIterations + 1

  override def fit(trainingFeatures: RDD[SparseVector[Double]], trainingLabels: RDD[DenseVector[Double]]): SparseLinearMapper = {
    val world = job.world
    val (d, k) = (trainingFeatures.first().length, trainingLabels.first().length)   // a rank may hold no rows
    val zipped = trainingFeatures.zip(trainingLabels).coalesce(world)
    val (fi, m, tol, it, lam, jb) = (fitIntercept, numCorrections, convergenceTol, numIterations, regParam, job)
    val models = zipped.barrier().mapPartitions { rowsIt =>
      val tc = org.apache.spark.BarrierTaskContext.get()
      val rank = tc.partitionId()
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(rank), rank, jb.world, jb.ncclId)
      val rows = rowsIt.toArray
      // CSR of this partition: SparseVector.activeSize entries per row, in storage order
      val indptr = new Array[Long](rows.length + 1)
      var q = 0
      while (q < rows.length) { indptr(q + 1) = indptr(q) + rows(q)._1.activeSize; q += 1 }
      val indices = new Array[Int](indptr(rows.length).toInt)
      val values = new Array[Double](indices.length)
      q = 0
      while (q < rows.length) {
        val v = rows(q)._1
        System.arraycopy(v.index, 0, indices, indptr(q).toInt, v.activeSize)
        System.arraycopy(v.data, 0, values, indptr(q).toInt, v.activeSize)
        q += 1
      }
      val s = lib.sparseFromHostCsr(c, indptr, indices, values, d)
      val y = lib.matrixCreate(c, rows.length, k)
      if (rows.nonEmpty) lib.matrixWriteRows(c, y, 0, GpuExecutor.flatten(rows.map(_._2)), rows.length, k)
      tc.barrier()
      val h = lib.sparseLbfgsFit(c, s, y, fi, m, tol, it, lam)                 // collective: NCCL all-reduce of A^T R inside
      val out = if (rank == 0) {
        val nb = lib.modelNumBlocks(c, h)
        Iterator.single(((0 until nb).map(j => lib.modelGetBlock(c, h, j)).toArray, if (fi) lib.modelGetIntercept(c, h) else null, k))
      } else Iterator.empty
      lib.modelDestroy(c, h); lib.sparseDestroy(c, s); lib.matrixDestroy(c, y)
      out
    }.collect()
    val (ws, b, _) = models.head
    val x = DenseMatrix.vertcat(ws.map(w => new DenseMatrix[Double](w.length / k, k, w)): _*)   // feature blocks, in order
    new SparseLinearMapper(x, if (fitIntercept) Some(DenseVector(b)) else None)
  }
}
