package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.workflow.{LabelEstimator, Transformer}
import org.apache.spark.broadcast.Broadcast
import org.apache.spark.rdd.RDD

import scala.util.Random

/**
 * Drop-in for keystoneml.nodes.learning.KernelRidgeRegression with a GaussianKernelGenerator(gamma)
 * (KernelRidgeRegression.scala:37-84, KernelGenerator.scala:36-194): same hyper-parameters, same block Gauss-Seidel over
 * contiguous blocks of training rows.  Training rows and labels are coalesced to one partition group per GPU; every executor
 * uploads ITS rows, ks_gaussian_kernel_create gathers the training rows onto every GPU (collective) and ks_krr_fit runs the
 * epochs (collective; the K_B^T W reduction that replaces treeReduce is an NCCL all-reduce inside the call).  Rank 0 returns the
 * model blocks.  blockPermuter: a seed drawing one permutation of the blocks per epoch (scala.util.Random; the Python binding
 * uses numpy's PCG64, so the two bindings visit blocks in different orders for the same seed).  blocksBeforeCheckpoint has no
 * effect.  Not compiled in the build image (no JVM).
 */
class GpuKernelRidgeRegression(gamma: Double, lambda: Double, blockSize: Int, numEpochs: Int, blockPermuter: Option[Long] = None,
    blocksBeforeCheckpoint: Int = 25, job: GpuJob)
  extends LabelEstimator[DenseVector[Double], DenseVector[Double], DenseVector[Double]] {

  require(gamma > 0 && !gamma.isInfinite, "gamma must be finite and > 0")
  require(blockSize >= 1 && numEpochs >= 1, "blockSize and numEpochs must be >= 1")

  override def fit(data: RDD[DenseVector[Double]], labels: RDD[DenseVector[Double]]): GpuKernelBlockLinearMapper = {
    val world = job.world
    val zipped = data.zip(labels).coalesce(world)                                // one partition per GPU, in partition order
    val nTrain = zipped.count()
    val nb = ((nTrain + blockSize - 1) / blockSize).toInt
    val order = blockPermuter.map { seed =>
      val rnd = new Random(seed)
      (0 until numEpochs).flatMap(_ => rnd.shuffle((0 until nb).toIndexedSeq)).toArray
    }.orNull
    val (g, lam, bs, ne, jb) = (gamma, lambda, blockSize, numEpochs, job)
    val models = zipped.barrier().mapPartitions { it =>
      val tc = org.apache.spark.BarrierTaskContext.get()
      val rank = tc.partitionId()
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(rank), rank, jb.world, jb.ncclId)
      val rows = it.toArray
      val d = if (rows.isEmpty) 0 else rows(0)._1.length
      val k = if (rows.isEmpty) 0 else rows(0)._2.length
      val x = lib.matrixCreate(c, rows.length, d)
      val y = lib.matrixCreate(c, rows.length, k)
      if (rows.nonEmpty) {
        lib.matrixWriteRows(c, x, 0, GpuExecutor.flatten(rows.map(_._1)), rows.length, d)
        lib.matrixWriteRows(c, y, 0, GpuExecutor.flatten(rows.map(_._2)), rows.length, k)
      }
      tc.barrier()
      val kern = lib.gaussianKernelCreate(c, x, g)                                // collective: all training rows on every GPU
      val m = lib.krrFit(c, kern, y, lam, bs, ne, order)                          // collective
      val out = if (rank == 0) {
        val nbm = lib.modelNumBlocks(c, m)
        Iterator.single(((0 until nbm).map(j => lib.modelGetBlock(c, m, j)).toArray, k))
      } else Iterator.empty
      lib.modelDestroy(c, m); lib.gaussianKernelDestroy(c, kern); lib.matrixDestroy(c, x); lib.matrixDestroy(c, y)
      out
    }.collect()
    val (ws, k) = models.head
    val xs = ws.map(w => new DenseMatrix[Double](w.length / k, k, w)).toSeq
    // apply needs the training rows in the fit's order (partition order of the coalesced RDD)
    val trainRows = data.sparkContext.broadcast(zipped.map(_._1).collect())
    new GpuKernelBlockLinearMapper(xs, blockSize, gamma, trainRows, job)
  }
}

/**
 * KernelBlockLinearMapper (KernelBlockLinearMapper.scala:28-89) on the GPU: sum_j K(x, X_j) W_j.  Each executor builds the
 * kernel object from the broadcast training rows once per batch (world 1 per executor context here: the rows are all local),
 * rebuilds the model (ks_kernel_model_from_host) and applies it to its partition.  Kernel models are not persisted.
 */
class GpuKernelBlockLinearMapper(val xs: Seq[DenseMatrix[Double]], val blockSize: Int, gamma: Double,
    trainRows: Broadcast[Array[DenseVector[Double]]], job: GpuJob) extends Transformer[DenseVector[Double], DenseVector[Double]] {
  private val xsData = xs.map(_.data).toArray
  private val k = xs.head.cols

  override def apply(in: RDD[DenseVector[Double]]): RDD[DenseVector[Double]] = {
    val (kk, bs, g, jb, tr, w) = (k, blockSize, gamma, job, trainRows, xsData)
    in.mapPartitionsWithIndex { case (p, it) =>
      val rows = it.toArray
      if (rows.isEmpty) Iterator.empty
      else {
        val lib = GpuExecutor.lib
        val rank = p % jb.world
        val c = GpuExecutor.ctx(jb.deviceOf(rank), rank, 1, null)
        val train = tr.value
        val xt = lib.matrixCreate(c, train.length, train(0).length)
        lib.matrixWriteRows(c, xt, 0, GpuExecutor.flatten(train), train.length, train(0).length)
        val kern = lib.gaussianKernelCreate(c, xt, g)
        val m = lib.kernelModelFromHost(c, kern, w, kk, bs)
        val x = lib.matrixCreate(c, rows.length, rows(0).length)
        lib.matrixWriteRows(c, x, 0, GpuExecutor.flatten(rows), rows.length, rows(0).length)
        try {
          val y = lib.modelApply(c, m, x, 0L, null)
          val flat = lib.matrixToHost(c, y)
          lib.matrixDestroy(c, y)
          Iterator.tabulate(rows.length)(i => DenseVector(java.util.Arrays.copyOfRange(flat, i * kk, (i + 1) * kk)))
        } finally {
          lib.modelDestroy(c, m); lib.gaussianKernelDestroy(c, kern); lib.matrixDestroy(c, x); lib.matrixDestroy(c, xt)
        }
      }
    }
  }

  override def apply(in: DenseVector[Double]): DenseVector[Double] = {
    val train = trainRows.value
    val out = DenseVector.zeros[Double](k)
    var j = 0
    var r0 = 0
    while (r0 < train.length) {
      val r1 = math.min(train.length, r0 + blockSize)
      val kv = DenseVector.tabulate(r1 - r0) { i => val df = train(r0 + i) - in; math.exp(-gamma * (df dot df)) }
      out += xs(j).t * kv
      j += 1
      r0 = r1
    }
    out
  }
}
