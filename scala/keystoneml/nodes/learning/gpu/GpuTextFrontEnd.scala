package keystoneml.nodes.learning.gpu

import breeze.linalg.SparseVector
import keystoneml.nodes.util.SparseFeatureVectorizer
import keystoneml.workflow.{Estimator, Transformer}
import org.apache.spark.rdd.RDD

import java.nio.charset.StandardCharsets

/**
 * The text front end of K/pipelines/text/{AmazonReviewsPipeline,NewsgroupsPipeline}.scala on the GPU (DESIGN.md section 23):
 *
 *   Trim andThen LowerCase() andThen Tokenizer() andThen NGramsFeaturizer(orders) andThen TermFrequency(fun)
 *     andThen (CommonSparseFeatures(numFeatures), train)                      -> GpuCommonSparseFeatures(...).fit(train)
 *   ... andThen NGramsFeaturizer(orders) andThen HashingTF(numFeatures)       -> GpuNGramsHashingTF(orders, numFeatures)
 *
 * Each executor uploads its partition's strings as UTF-8 and runs every step from the bytes to the CSR on its device (ks_text_*,
 * ks_term_frequency, ks_sparse_features_*, ks_hashing_tf); rows come back as Breeze SparseVectors (columns ascending, fp64).  The
 * vocabulary fit runs on one partition (an exact top-K over ranks is not implemented), as CommonSparseFeatures' semantics of §23
 * require; on an executor whose context was created for a multi-rank job the library refuses that fit.  Not compiled in the build
 * image (no JVM).
 */
private[gpu] object GpuText {
  final val Trim = 1       // KS_TEXT_TRIM
  final val Lower = 2      // KS_TEXT_LOWER
  final val TermFirst = 5  // KS_TEXT_TERM_FIRST
  final val TermOrder = 6  // KS_TEXT_TERM_ORDER
  final val Bytes = 0      // KS_TEXT_BYTES
  final val TokenBegin = 2 // KS_TEXT_TOKEN_BEGIN
  final val TokenEnd = 3   // KS_TEXT_TOKEN_END

  def utf8(strings: Array[String]): (Array[Byte], Array[Long]) = {
    val parts = strings.map(_.getBytes(StandardCharsets.UTF_8))
    val off = new Array[Long](parts.length + 1)
    var i = 0
    while (i < parts.length) { off(i + 1) = off(i) + parts(i).length; i += 1 }
    val bytes = new Array[Byte](off(parts.length).toInt)
    i = 0
    while (i < parts.length) { System.arraycopy(parts(i), 0, bytes, off(i).toInt, parts(i).length); i += 1 }
    (bytes, off)
  }

  /** Trim, LowerCase, Tokenizer, the n-grams of orders (minOrder to maxOrder; 0, 0 = the tokens) and TermFrequency(fun) of docs:
   *  the term-frequency handle; the caller releases it with textDestroy. */
  def termFrequencies(lib: KeystoneB200, c: Long, docs: Array[String], minOrder: Int, maxOrder: Int, fun: Double => Double): Long = {
    val (bytes, off) = utf8(docs)
    val text = lib.textFromHost(c, bytes, off)
    val trimmed = lib.textTransform(c, text, Trim)
    val lowered = lib.textTransform(c, trimmed, Lower)
    val tokens = lib.textTokenize(c, lowered)
    val Array(tf, maxCount) = lib.termFrequency(c, tokens, minOrder, maxOrder)
    if (maxCount > 0) lib.tfSetWeights(c, tf, Array.tabulate(maxCount.toInt)(i => fun((i + 1).toDouble)))
    Seq(tokens, lowered, trimmed, text).foreach(h => lib.textDestroy(c, h))   // tf keeps what it needs alive
    tf
  }

  def rows(lib: KeystoneB200, c: Long, s: Long, numCols: Int): Iterator[SparseVector[Double]] = {
    val csr = lib.sparseToHostCsr(c, s)
    lib.sparseDestroy(c, s)
    val indptr = csr(0).asInstanceOf[Array[Long]]
    val indices = csr(1).asInstanceOf[Array[Int]]
    val values = csr(2).asInstanceOf[Array[Double]]
    Iterator.tabulate(indptr.length - 1) { r =>
      val (a, b) = (indptr(r).toInt, indptr(r + 1).toInt)
      new SparseVector[Double](indices.slice(a, b), values.slice(a, b), numCols)
    }
  }

  /** The feature space of a space handle as the reference's Map[Seq[String], Int] (n-grams; a plain token becomes a Seq of one). */
  def featureSpace(lib: KeystoneB200, c: Long, space: Long): Map[Seq[String], Int] = {
    val bytes = lib.textArrayBytes(c, space, Bytes)
    val tb = lib.textArrayLongs(c, space, TokenBegin)
    val te = lib.textArrayLongs(c, space, TokenEnd)
    val first = lib.textArrayLongs(c, space, TermFirst)
    val order = lib.textArrayInts(c, space, TermOrder)
    val tok = Array.tabulate(tb.length)(t => new String(bytes, tb(t).toInt, (te(t) - tb(t)).toInt, StandardCharsets.UTF_8))
    first.indices.map(f => (tok.slice(first(f).toInt, first(f).toInt + math.max(order(f), 1)).toSeq, f)).toMap
  }
}

/**
 * The text pipelines' featurizer and CommonSparseFeatures(numFeatures).fit on raw strings: Trim, LowerCase, Tokenizer,
 * NGramsFeaturizer(orders) (consecutive, 1 to 4) and TermFrequency(fun), then the most frequent n-grams by document frequency, ties by
 * earliest appearance.  The fit gathers the training strings into one partition.  Returns a GpuTextVectorizer, whose
 * `vectorizer` is the reference's SparseFeatureVectorizer over the same space.
 */
case class GpuCommonSparseFeatures(numFeatures: Int, orders: Seq[Int], fun: Double => Double, job: GpuJob)
    extends Estimator[String, SparseVector[Double]] {
  require(orders.nonEmpty && orders.min >= 1 && orders.max <= 4 && orders.sliding(2).forall(p => p.length < 2 || p(1) == p(0) + 1),
    "orders must be consecutive, >= 1 and <= 4")

  override def fit(data: RDD[String]): GpuTextVectorizer = {
    val (mn, mx, k, f, jb) = (orders.min, orders.max, numFeatures, fun, job)
    val space = data.coalesce(1).mapPartitions { it =>
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(0), 0, 1, null)
      val tf = GpuText.termFrequencies(lib, c, it.toArray, mn, mx, f)
      val sp = lib.sparseFeaturesFit(c, tf, k)
      val out = GpuText.featureSpace(lib, c, sp)
      lib.textDestroy(c, sp)
      lib.textDestroy(c, tf)
      Iterator.single(out)
    }.collect().head
    GpuTextVectorizer(space, orders, fun, job)
  }
}

/** SparseFeatureVectorizer(featureSpace) applied to the n-gram term frequencies of raw strings, per partition on the device. */
case class GpuTextVectorizer(featureSpace: Map[Seq[String], Int], orders: Seq[Int], fun: Double => Double, job: GpuJob)
    extends Transformer[String, SparseVector[Double]] {
  def vectorizer: SparseFeatureVectorizer[Seq[String]] = new SparseFeatureVectorizer(featureSpace)

  override def apply(in: String): SparseVector[Double] = vectorizer.apply(
    keystoneml.nodes.stats.TermFrequency(fun).apply(keystoneml.nodes.nlp.NGramsFeaturizer[String](orders).apply(
      keystoneml.nodes.nlp.Tokenizer().apply(keystoneml.nodes.nlp.LowerCase().apply(keystoneml.nodes.nlp.Trim.apply(in))))))

  override def apply(in: RDD[String]): RDD[SparseVector[Double]] = {
    val (mn, mx, f, jb, n) = (orders.min, orders.max, fun, job, featureSpace.size)
    val terms = featureSpace.toSeq.sortBy(_._2).map(_._1).toArray
    in.mapPartitionsWithIndex { (p, it) =>
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(p % jb.world), 0, 1, null)
      val docs = it.toArray
      val first = new Array[Long](terms.length)
      val order = terms.map(_.length)
      var q = 0
      while (q < terms.length - 1) { first(q + 1) = first(q) + terms(q).length; q += 1 }
      val (bytes, toff) = GpuText.utf8(terms.flatten)
      val tokens = lib.tokensFromHost(c, bytes, toff, Array(0L, toff.length - 1L))
      val space = lib.sparseFeaturesFromHost(c, tokens, first, order)
      val tf = GpuText.termFrequencies(lib, c, docs, mn, mx, f)
      val s = lib.sparseFeaturesApply(c, space, tf)
      Seq(tf, space, tokens).foreach(h => lib.textDestroy(c, h))
      GpuText.rows(lib, c, s, n)
    }
  }
}

/** NGramsHashingTF(orders, numFeatures) (K/nodes/nlp/NGramsHashingTF.scala) on token sequences, per partition on the device. */
case class GpuNGramsHashingTF(orders: Seq[Int], numFeatures: Int, job: GpuJob) extends Transformer[Seq[String], SparseVector[Double]] {
  override def apply(in: Seq[String]): SparseVector[Double] = keystoneml.nodes.nlp.NGramsHashingTF(orders, numFeatures).apply(in)

  override def apply(in: RDD[Seq[String]]): RDD[SparseVector[Double]] = {
    val (mn, mx, nf, jb) = (orders.min, orders.max, numFeatures, job)
    in.mapPartitionsWithIndex { (p, it) =>
      val lib = GpuExecutor.lib
      val c = GpuExecutor.ctx(jb.deviceOf(p % jb.world), 0, 1, null)
      val docs = it.toArray
      val doff = docs.scanLeft(0L)(_ + _.length)
      val (bytes, toff) = GpuText.utf8(docs.flatten)
      val tokens = lib.tokensFromHost(c, bytes, toff, doff)
      val s = lib.hashingTf(c, tokens, mn, mx, nf)
      lib.textDestroy(c, tokens)
      GpuText.rows(lib, c, s, nf)
    }
  }
}
