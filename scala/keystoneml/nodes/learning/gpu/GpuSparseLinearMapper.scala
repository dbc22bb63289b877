package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.nodes.learning.SparseLinearMapper
import keystoneml.workflow.Transformer
import org.apache.spark.rdd.RDD

/**
 * SparseLinearMapper.apply on the GPU (K/nodes/learning/SparseLinearMapper.scala): wraps a fitted reference-side mapper (x, bOpt),
 * rebuilds the model on each executor's context once per partition (ks_model_from_host, feature blocks of min(d, 4096) rows),
 * uploads the partition's SparseVectors as CSR and maps them through ks_model_apply_sparse (A x + b in fp64, rounded once to fp32).
 * Not compiled in the build image (no JVM).
 */
class GpuSparseLinearMapper(mapper: SparseLinearMapper, job: GpuJob) extends Transformer[SparseVector[Double], DenseVector[Double]] {
  private val d = mapper.x.rows
  private val k = mapper.x.cols
  private val blockSize = math.min(d, 4096)
  private val xsData = (0 until d by blockSize).map(r0 => mapper.x(r0 until math.min(d, r0 + blockSize), ::).copy.data).toArray
  private val b = mapper.bOpt.map(_.data).orNull

  override def apply(in: RDD[SparseVector[Double]]): RDD[DenseVector[Double]] = {
    val (kk, dd, bs, xs, bb) = (k, d, blockSize, xsData, b)
    in.mapPartitionsWithIndex { case (p, it) =>
      val rows = it.toArray
      if (rows.isEmpty) Iterator.empty
      else {
        val lib = GpuExecutor.lib
        val rank = p % job.world
        val c = GpuExecutor.ctx(job.deviceOf(rank), rank, 1, null)
        val indptr = new Array[Long](rows.length + 1)
        for (q <- rows.indices) indptr(q + 1) = indptr(q) + rows(q).activeSize
        val indices = new Array[Int](indptr(rows.length).toInt)
        val values = new Array[Double](indices.length)
        for (q <- rows.indices) {
          System.arraycopy(rows(q).index, 0, indices, indptr(q).toInt, rows(q).activeSize)
          System.arraycopy(rows(q).data, 0, values, indptr(q).toInt, rows(q).activeSize)
        }
        val s = lib.sparseFromHostCsr(c, indptr, indices, values, dd)
        val m = lib.modelFromHost(c, xs, bs, kk, bb, null)
        try {
          val y = lib.modelApplySparse(c, m, s)
          val flat = lib.matrixToHost(c, y)
          lib.matrixDestroy(c, y)
          Iterator.tabulate(rows.length)(i => DenseVector(java.util.Arrays.copyOfRange(flat, i * kk, (i + 1) * kk)))
        } finally { lib.modelDestroy(c, m); lib.sparseDestroy(c, s) }
      }
    }
  }

  override def apply(in: SparseVector[Double]): DenseVector[Double] = mapper.apply(in)  // single datum: the JVM path
}
