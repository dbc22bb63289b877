package keystoneml.nodes.learning.gpu

import breeze.linalg._
import org.apache.spark.rdd.RDD

/**
 * The barrier stage shared by GpuLogisticRegressionEstimator and GpuNaiveBayesEstimator: each executor uploads its partition's rows
 * (SparseVectors as CSR through ks_sparse_from_host_csr, other vectors as dense rows), runs the collective fit given as `fit`
 * (ctx, features handle or 0, sparse handle or 0, class ids) and rank 0 returns the model's feature blocks (column-major, d x k in
 * blocks of min(d, 4096) rows) and its intercept.  Not compiled in the build image (no JVM).
 */
private[gpu] object GpuClassifierFit {
  def apply[T <: Vector[Double]](in: RDD[T], labels: RDD[Int], job: GpuJob,
      fit: (KeystoneB200, Long, Long, Long, Array[Int]) => Long): (DenseMatrix[Double], Array[Double]) = {
    val d = in.first().length   // a rank may hold no rows
    val zipped = in.zip(labels).coalesce(job.world)
    val jb = job
    val models = zipped.barrier().mapPartitions { rowsIt =>
      val tc = org.apache.spark.BarrierTaskContext.get()
      val rank = tc.partitionId()
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(rank), rank, jb.world, jb.ncclId)
      val rows = rowsIt.toArray
      val classes = rows.map(_._2)
      val sparse = rows.headOption.exists(_._1.isInstanceOf[SparseVector[_]])
      val (f, s) = if (sparse) {
        val indptr = new Array[Long](rows.length + 1)
        var q = 0
        while (q < rows.length) { indptr(q + 1) = indptr(q) + rows(q)._1.asInstanceOf[SparseVector[Double]].activeSize; q += 1 }
        val indices = new Array[Int](indptr(rows.length).toInt)
        val values = new Array[Double](indices.length)
        q = 0
        while (q < rows.length) {
          val v = rows(q)._1.asInstanceOf[SparseVector[Double]]
          System.arraycopy(v.index, 0, indices, indptr(q).toInt, v.activeSize)
          System.arraycopy(v.data, 0, values, indptr(q).toInt, v.activeSize)
          q += 1
        }
        (0L, lib.sparseFromHostCsr(c, indptr, indices, values, d))
      } else {
        val m = lib.matrixCreate(c, rows.length, d)
        if (rows.nonEmpty) lib.matrixWriteRows(c, m, 0, GpuExecutor.flatten(rows.map(_._1.toDenseVector)), rows.length, d)
        (m, 0L)
      }
      tc.barrier()
      val h = fit(lib, c, f, s, classes)                 // collective: NCCL all-reduces inside
      val out = if (rank == 0) {
        val nb = lib.modelNumBlocks(c, h)
        Iterator.single(((0 until nb).map(j => lib.modelGetBlock(c, h, j)).toArray, lib.modelGetIntercept(c, h)))
      } else Iterator.empty
      lib.modelDestroy(c, h)
      if (s != 0L) lib.sparseDestroy(c, s) else lib.matrixDestroy(c, f)
      out
    }.collect()
    val (ws, b) = models.head
    val k = b.length
    (DenseMatrix.vertcat(ws.map(w => new DenseMatrix[Double](w.length / k, k, w)): _*), b)
  }
}
