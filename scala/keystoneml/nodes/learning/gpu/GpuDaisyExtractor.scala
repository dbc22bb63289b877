package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.utils.Image
import keystoneml.workflow.Transformer
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.images.DaisyExtractor(daisyT, daisyQ, daisyR, daisyH, pixelBorder, stride, patchSize) on a
 * one-channel (GrayScaler) image: the same daisyFeatureSize x nKP Float matrix per image, computed on this executor's GPU
 * (DESIGN.md section 19).  patchSize is unused, as in the reference.  The RDD apply sends each partition's images to the device in
 * batches of equal shape (one ks_daisy_extract per batch).  Not collective.  Not compiled in the build image (no JVM).
 */
class GpuDaisyExtractor(val daisyT: Int = 8, val daisyQ: Int = 3, val daisyR: Int = 7, val daisyH: Int = 8, val pixelBorder: Int = 16,
    val stride: Int = 4, val patchSize: Int = 24, job: GpuJob)
  extends Transformer[Image, DenseMatrix[Float]] {

  val daisyFeatureSize = daisyH * (daisyT * daisyQ + 1)

  /** One-channel ImageVectorizer order: value (x, y) at x + y * xDim. */
  private def vectorize(im: Image, out: Array[Double], off: Int): Unit = {
    require(im.metadata.numChannels == 1, "GpuDaisyExtractor needs one-channel images (apply GrayScaler first)")
    val (xd, yd) = (im.metadata.xDim, im.metadata.yDim)
    var y = 0
    while (y < yd) { var x = 0
      while (x < xd) { out(off + x + y * xd) = im.get(x, y, 0).toFloat; x += 1 }
      y += 1 }
  }

  /** One device call for images of one shape; returns one descriptor matrix per image. */
  def applyBatch(images: Array[Image]): Array[DenseMatrix[Float]] = {
    val lib = GpuExecutor.lib
    val c = GpuExecutor.ctx(job.deviceOf(0), 0, 1, null)
    val md = images(0).metadata
    val px = md.xDim * md.yDim
    val flat = new Array[Double](images.length * px)
    images.zipWithIndex.foreach { case (im, i) => vectorize(im, flat, i * px) }
    val m = lib.matrixCreate(c, images.length, px)
    lib.matrixWriteRows(c, m, 0, flat, images.length, px)
    val d = lib.daisyExtract(c, m, md.xDim, md.yDim, daisyT, daisyQ, daisyR, daisyH, pixelBorder, stride)
    val host = lib.matrixToHost(c, d)   // (n nKP) x daisyFeatureSize row-major: image i's rows are its matrix, column-major
    lib.matrixDestroy(c, d); lib.matrixDestroy(c, m)
    val per = host.length / images.length
    images.indices.map { i =>
      new DenseMatrix[Double](daisyFeatureSize, per / daisyFeatureSize, host.slice(i * per, (i + 1) * per)).map(_.toFloat)
    }.toArray
  }

  override def apply(image: Image): DenseMatrix[Float] = applyBatch(Array(image))(0)

  override def apply(in: RDD[Image]): RDD[DenseMatrix[Float]] = in.mapPartitions { it =>
    val images = it.toArray
    val out = new Array[DenseMatrix[Float]](images.length)
    images.indices.groupBy(i => (images(i).metadata.xDim, images(i).metadata.yDim)).values.foreach { idx =>
      applyBatch(idx.map(images).toArray).zip(idx).foreach { case (m, i) => out(i) = m }
    }
    out.iterator
  }
}
