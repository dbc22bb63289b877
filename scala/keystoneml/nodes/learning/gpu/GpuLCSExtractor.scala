package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.utils.Image
import keystoneml.workflow.Transformer
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.images.LCSExtractor(stride, strideStart, subPatchSize): the same (n^2 C 2) x nKP Float descriptor
 * matrix per image, computed on this executor's GPU (window statistics in fp64, rounded once to fp32; DESIGN.md section 16).
 * The RDD apply sends each partition's images to the device in batches of equal shape (one ks_lcs_extract per batch).  Not
 * collective.  Not compiled in the build image (no JVM).
 */
class GpuLCSExtractor(val stride: Int, val strideStart: Int, val subPatchSize: Int, job: GpuJob)
  extends Transformer[Image, DenseMatrix[Float]] {

  /** ImageVectorizer order: value (x, y, c) at c + x * C + y * C * xDim. */
  private def vectorize(im: Image, out: Array[Double], off: Int): Unit = {
    val (xd, yd, nc) = (im.metadata.xDim, im.metadata.yDim, im.metadata.numChannels)
    var y = 0
    while (y < yd) { var x = 0
      while (x < xd) { var c = 0
        while (c < nc) { out(off + c + x * nc + y * nc * xd) = im.get(x, y, c); c += 1 }
        x += 1 }
      y += 1 }
  }

  /** One device call for images of one shape; returns one descriptor matrix per image. */
  def applyBatch(images: Array[Image]): Array[DenseMatrix[Float]] = {
    val lib = GpuExecutor.lib
    val c = GpuExecutor.ctx(job.deviceOf(0), 0, 1, null)
    val md = images(0).metadata
    val px = md.xDim * md.yDim * md.numChannels
    val flat = new Array[Double](images.length * px)
    images.zipWithIndex.foreach { case (im, i) => vectorize(im, flat, i * px) }
    val m = lib.matrixCreate(c, images.length, px)
    lib.matrixWriteRows(c, m, 0, flat, images.length, px)
    val d = lib.lcsExtract(c, m, md.xDim, md.yDim, md.numChannels, stride, strideStart, subPatchSize)
    val host = lib.matrixToHost(c, d)   // (n nKP) x dim row-major: image i's rows are its dim x nKP matrix, column-major
    lib.matrixDestroy(c, d); lib.matrixDestroy(c, m)
    val dim = 4 * 4 * md.numChannels * 2   // 4 neighbours per axis for every subPatchSize, (mean, std) per channel
    val per = host.length / images.length
    images.indices.map { i => new DenseMatrix[Double](dim, per / dim, host.slice(i * per, (i + 1) * per)).map(_.toFloat) }.toArray
  }

  override def apply(image: Image): DenseMatrix[Float] = applyBatch(Array(image))(0)

  override def apply(in: RDD[Image]): RDD[DenseMatrix[Float]] = in.mapPartitions { it =>
    val images = it.toArray
    val out = new Array[DenseMatrix[Float]](images.length)
    images.indices.groupBy(i => (images(i).metadata.xDim, images(i).metadata.yDim, images(i).metadata.numChannels)).values.foreach { idx =>
      applyBatch(idx.map(images).toArray).zip(idx).foreach { case (m, i) => out(i) = m }
    }
    out.iterator
  }
}
