package keystoneml.nodes.learning.gpu

import breeze.linalg._
import keystoneml.utils.Image
import keystoneml.workflow.Transformer
import org.apache.spark.rdd.RDD

/**
 * Drop-in for keystoneml.nodes.images.HogExtractor(binSize) on a three-channel BGR image: the same (cells x 32) Float matrix per
 * image, row y + x (nY - 2), computed on this executor's GPU (DESIGN.md section 19).  With pixelScale = true the images are the
 * PixelScaler's input and the device takes x / 255.0 in fp64, as the reference's mapPixels does; apply it to unscaled images then.
 * The RDD apply sends each partition's images to the device in batches of equal shape (one ks_hog_extract per batch).  Not
 * collective.  Not compiled in the build image (no JVM).
 */
class GpuHogExtractor(val binSize: Int, val pixelScale: Boolean = false, job: GpuJob)
  extends Transformer[Image, DenseMatrix[Float]] {

  val numFeatures = 32

  /** ImageVectorizer order: value (x, y, c) at c + x * C + y * C * xDim. */
  private def vectorize(im: Image, out: Array[Double], off: Int): Unit = {
    require(im.metadata.numChannels == 3, "GpuHogExtractor needs three-channel (BGR) images")
    val (xd, yd) = (im.metadata.xDim, im.metadata.yDim)
    var y = 0
    while (y < yd) { var x = 0
      while (x < xd) { var c = 0
        while (c < 3) { out(off + c + x * 3 + y * 3 * xd) = im.get(x, y, c).toFloat; c += 1 }
        x += 1 }
      y += 1 }
  }

  /** One device call for images of one shape; returns one feature matrix per image. */
  def applyBatch(images: Array[Image]): Array[DenseMatrix[Float]] = {
    val lib = GpuExecutor.lib
    val c = GpuExecutor.ctx(job.deviceOf(0), 0, 1, null)
    val md = images(0).metadata
    val px = md.xDim * md.yDim * 3
    val flat = new Array[Double](images.length * px)
    images.zipWithIndex.foreach { case (im, i) => vectorize(im, flat, i * px) }
    val m = lib.matrixCreate(c, images.length, px)
    lib.matrixWriteRows(c, m, 0, flat, images.length, px)
    val d = lib.hogExtract(c, m, md.xDim, md.yDim, 3, if (pixelScale) 1 else 0, binSize)
    val host = lib.matrixToHost(c, d)   // (n cells) x 32 row-major
    lib.matrixDestroy(c, d); lib.matrixDestroy(c, m)
    val per = host.length / images.length
    images.indices.map { i =>
      new DenseMatrix[Double](numFeatures, per / numFeatures, host.slice(i * per, (i + 1) * per)).t.copy.map(_.toFloat)
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
