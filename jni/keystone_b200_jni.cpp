// JNI shim: 1:1 wrappers from keystoneml.nodes.learning.gpu.KeystoneB200 (scala/.../KeystoneB200.scala) to the C ABI
// (include/keystone_b200.h).  Follows the reference's own native convention -- a Serializable Scala class whose
// constructor calls System.loadLibrary, @native methods taking only primitives / primitive arrays
// (/root/reference/src/main/scala/keystoneml/utils/external/VLFeat.scala:18-26, src/main/cpp/VLFeat.cxx:203-292) -- but
// errors become RuntimeExceptions instead of exit(-1) (src/main/cpp/EncEval.cxx:43-47).
//
// Rules kept throughout: (1) after a failed call the wrapper throws and RETURNS AT ONCE -- no JNI call is made with an
// exception pending; (2) no Get/ReleasePrimitiveArrayCritical around CUDA work (a critical region blocks the collector while
// cudaMemcpy / stream synchronisation wait): inputs are pinned or copied with Get<Type>ArrayElements, outputs are written with
// Set<Type>ArrayRegion from the model's pinned host mirror.
//
// NOT COMPILED IN THIS IMAGE: there is no JDK (no jni.h).  Build where one exists:
//   g++ -O2 -fPIC -shared -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude jni/keystone_b200_jni.cpp \
//       -Lkeystone_b200/lib -lkeystone_b200 -o lib/libkeystone_b200_jni.so
#include <jni.h>

#include <vector>

#include "keystone_b200.h"

#define JFN(ret, name) extern "C" JNIEXPORT ret JNICALL Java_keystoneml_nodes_learning_gpu_KeystoneB200_##name

// true = OK; false = a RuntimeException is now pending and the caller must return immediately
static bool ok(JNIEnv* env, jlong ctx, int32_t rc) {
  if (rc == KS_OK) return true;
  jclass ex = env->FindClass("java/lang/RuntimeException");
  if (ex) env->ThrowNew(ex, ks_last_error(ctx));
  return false;
}

struct LongArray {  // borrowed view of a jlongArray (may be null)
  JNIEnv* env;
  jlongArray arr;
  jlong* p = nullptr;
  jsize n = 0;
  LongArray(JNIEnv* e, jlongArray a) : env(e), arr(a) {
    if (arr) {
      n = env->GetArrayLength(arr);
      if (n) p = env->GetLongArrayElements(arr, nullptr);
    }
  }
  ~LongArray() {
    if (p) env->ReleaseLongArrayElements(arr, p, JNI_ABORT);
  }
  const int64_t* data() const { return reinterpret_cast<const int64_t*>(p); }
};

JFN(jbyteArray, ncclUniqueId)(JNIEnv* env, jobject) {
  uint8_t id[KS_NCCL_ID_BYTES];
  if (!ok(env, 0, ks_nccl_unique_id(id))) return nullptr;
  jbyteArray out = env->NewByteArray(KS_NCCL_ID_BYTES);
  if (!out) return nullptr;
  env->SetByteArrayRegion(out, 0, KS_NCCL_ID_BYTES, reinterpret_cast<const jbyte*>(id));
  return out;
}

JFN(jlong, ctxCreate)(JNIEnv* env, jobject, jint device, jint rank, jint world, jbyteArray ncclId) {
  int64_t h = 0;
  jbyte* id = ncclId ? env->GetByteArrayElements(ncclId, nullptr) : nullptr;
  const int32_t rc = ks_ctx_create(device, rank, world, reinterpret_cast<const uint8_t*>(id), &h);
  if (id) env->ReleaseByteArrayElements(ncclId, id, JNI_ABORT);
  return ok(env, 0, rc) ? h : 0;
}
JFN(void, ctxDestroy)(JNIEnv*, jobject, jlong ctx) { ks_ctx_destroy(ctx); }
JFN(void, ctxSetOption)(JNIEnv* env, jobject, jlong ctx, jstring name, jlong value) {
  const char* s = env->GetStringUTFChars(name, nullptr);
  if (!s) return;
  const int32_t rc = ks_ctx_set_option(ctx, s, value);
  env->ReleaseStringUTFChars(name, s);
  ok(env, ctx, rc);
}

// ---- matrices: an executor creates one matrix for all its rows and writes one partition at a time
JFN(jlong, matrixCreate)(JNIEnv* env, jobject, jlong ctx, jlong nRows, jlong nCols) {
  int64_t h = 0;
  return ok(env, ctx, ks_matrix_create(ctx, nRows, nCols, &h)) ? h : 0;
}
// rows are one flat row-major double array (MatrixUtils.rowsToMatrix without the column-major transpose)
JFN(void, matrixWriteRows)(JNIEnv* env, jobject, jlong ctx, jlong m, jlong row0, jdoubleArray rowMajor, jlong nRows, jlong nCols) {
  jdouble* p = env->GetDoubleArrayElements(rowMajor, nullptr);
  if (!p) return;
  const int32_t rc = ks_matrix_write_rows_f64(ctx, m, row0, p, nRows, nCols);
  env->ReleaseDoubleArrayElements(rowMajor, p, JNI_ABORT);
  ok(env, ctx, rc);
}
JFN(jlong, labelsFromClasses)(JNIEnv* env, jobject, jlong ctx, jintArray classes, jint numClasses) {
  int64_t h = 0;
  const jsize n = env->GetArrayLength(classes);
  jint* p = env->GetIntArrayElements(classes, nullptr);
  if (!p) return 0;
  const int32_t rc = ks_labels_from_classes(ctx, reinterpret_cast<const int32_t*>(p), n, numClasses, &h);
  env->ReleaseIntArrayElements(classes, p, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jdoubleArray, matrixToHost)(JNIEnv* env, jobject, jlong ctx, jlong m) {
  int64_t r = 0, c = 0;
  if (!ok(env, ctx, ks_matrix_shape(ctx, m, &r, &c))) return nullptr;
  jdoubleArray out = env->NewDoubleArray(static_cast<jsize>(r * c));
  if (!out) return nullptr;
  jdouble* p = env->GetDoubleArrayElements(out, nullptr);
  if (!p) return nullptr;
  const int32_t rc = ks_matrix_to_host_f64(ctx, m, p, c);
  env->ReleaseDoubleArrayElements(out, p, 0);
  return ok(env, ctx, rc) ? out : nullptr;
}
JFN(void, matrixDestroy)(JNIEnv*, jobject, jlong ctx, jlong m) { ks_matrix_destroy(ctx, m); }

// ---- feature maps.  W = DenseMatrix.data (column-major numOut x numIn), b = DenseVector.data
JFN(jlong, cosineRfCreate)(JNIEnv* env, jobject, jlong ctx, jdoubleArray W, jdoubleArray b, jlong nOut, jlong nIn) {
  int64_t h = 0;
  jdouble* w = env->GetDoubleArrayElements(W, nullptr);
  if (!w) return 0;
  jdouble* bb = env->GetDoubleArrayElements(b, nullptr);
  if (!bb) {
    env->ReleaseDoubleArrayElements(W, w, JNI_ABORT);
    return 0;
  }
  const int32_t rc = ks_cosine_rf_create(ctx, w, bb, nOut, nIn, &h);
  env->ReleaseDoubleArrayElements(W, w, JNI_ABORT);
  env->ReleaseDoubleArrayElements(b, bb, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, paddedFftCreate)(JNIEnv* env, jobject, jlong ctx, jdoubleArray signs, jlong nIn, jboolean rectify, jdouble maxVal,
                            jdouble alpha) {
  int64_t h = 0;
  jdouble* s = signs ? env->GetDoubleArrayElements(signs, nullptr) : nullptr;
  const int32_t rc = ks_padded_fft_create(ctx, s, nIn, rectify ? 1 : 0, maxVal, alpha, &h);
  if (s) env->ReleaseDoubleArrayElements(signs, s, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, featureMapApply)(JNIEnv* env, jobject, jlong ctx, jlong rf, jlong xIn) {
  int64_t h = 0;
  return ok(env, ctx, ks_cosine_rf_apply(ctx, rf, xIn, &h)) ? h : 0;
}
JFN(void, featureMapDestroy)(JNIEnv*, jobject, jlong ctx, jlong rf) { ks_cosine_rf_destroy(ctx, rf); }

// ---- estimators (collective across the executors of the job)
JFN(jlong, blockLsFit)(JNIEnv* env, jobject, jlong ctx, jlong features, jlong xIn, jlongArray rfs, jlong labels, jint blockSize,
                       jint numIter, jdouble lambda, jlong numFeaturesOr0, jint precisionMode) {
  int64_t h = 0;
  LongArray r(env, rfs);
  const int32_t rc = ks_blockls_fit(ctx, features, xIn, r.data(), r.n, labels, blockSize, numIter, lambda, numFeaturesOr0,
                                    precisionMode, &h);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, blockWlsFit)(JNIEnv* env, jobject, jlong ctx, jlong features, jlong xIn, jlongArray rfs, jlong labels, jint blockSize,
                        jint numIter, jdouble lambda, jdouble mixtureWeight, jlong numFeaturesOr0, jint precisionMode) {
  int64_t h = 0;
  LongArray r(env, rfs);
  const int32_t rc = ks_blockwls_fit(ctx, features, xIn, r.data(), r.n, labels, blockSize, numIter, lambda, mixtureWeight,
                                     numFeaturesOr0, precisionMode, &h);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, lbfgsFit)(JNIEnv* env, jobject, jlong ctx, jlong features, jlong xIn, jlongArray rfs, jlong labels, jboolean fitIntercept,
                     jint numCorrections, jdouble convergenceTol, jint numIterations, jdouble regParam, jint precisionMode) {
  int64_t h = 0;
  LongArray r(env, rfs);
  const int32_t rc = ks_lbfgs_fit(ctx, features, xIn, r.data(), r.n, labels, fitIntercept ? 1 : 0, numCorrections, convergenceTol,
                                  numIterations, regParam, precisionMode, &h);
  return ok(env, ctx, rc) ? h : 0;
}
// ---- sparse matrices and SparseLBFGSwithL2 (DESIGN.md section 20)
JFN(jlong, sparseFromHostCsr)(JNIEnv* env, jobject, jlong ctx, jlongArray indptr, jintArray indices, jdoubleArray values, jlong nCols) {
  int64_t h = 0;
  const jsize nRows = env->GetArrayLength(indptr) - 1;
  const jsize nnz = env->GetArrayLength(indices);
  jlong* ip = env->GetLongArrayElements(indptr, nullptr);
  jint* ix = nnz ? env->GetIntArrayElements(indices, nullptr) : nullptr;
  jdouble* v = nnz ? env->GetDoubleArrayElements(values, nullptr) : nullptr;
  const int32_t rc = ks_sparse_from_host_csr(ctx, reinterpret_cast<const int64_t*>(ip), reinterpret_cast<const int32_t*>(ix), v, nRows,
                                             nCols, &h);
  if (v) env->ReleaseDoubleArrayElements(values, v, JNI_ABORT);
  if (ix) env->ReleaseIntArrayElements(indices, ix, JNI_ABORT);
  env->ReleaseLongArrayElements(indptr, ip, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(void, sparseDestroy)(JNIEnv*, jobject, jlong ctx, jlong s) { ks_sparse_destroy(ctx, s); }
JFN(jlong, sparseDensify)(JNIEnv* env, jobject, jlong ctx, jlong s) {
  int64_t h = 0;
  return ok(env, ctx, ks_sparse_densify(ctx, s, &h)) ? h : 0;
}
JFN(jlong, sparseLbfgsFit)(JNIEnv* env, jobject, jlong ctx, jlong s, jlong labels, jboolean fitIntercept, jint numCorrections,
                           jdouble convergenceTol, jint numIterations, jdouble regParam) {
  int64_t h = 0;
  const int32_t rc = ks_sparse_lbfgs_fit(ctx, s, labels, fitIntercept ? 1 : 0, numCorrections, convergenceTol, numIterations, regParam, &h);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, modelApplySparse)(JNIEnv* env, jobject, jlong ctx, jlong model, jlong s) {
  int64_t h = 0;
  return ok(env, ctx, ks_model_apply_sparse(ctx, model, s, &h)) ? h : 0;
}
// logistic regression / naive Bayes: exactly one of features and sparse is a handle; classes holds the partition's class ids
JFN(jlong, logisticFit)(JNIEnv* env, jobject, jlong ctx, jlong features, jlong sparse, jintArray classes, jint numClasses,
                        jdouble regParam, jint numIters, jdouble convergenceTol) {
  int64_t h = 0;
  const jsize n = classes ? env->GetArrayLength(classes) : 0;
  jint* p = n ? env->GetIntArrayElements(classes, nullptr) : nullptr;
  const int32_t rc = ks_logistic_fit(ctx, features, sparse, reinterpret_cast<const int32_t*>(p), n, numClasses, regParam, numIters,
                                     convergenceTol, &h);
  if (p) env->ReleaseIntArrayElements(classes, p, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, naiveBayesFit)(JNIEnv* env, jobject, jlong ctx, jlong features, jlong sparse, jintArray classes, jint numClasses,
                          jdouble lambda) {
  int64_t h = 0;
  const jsize n = classes ? env->GetArrayLength(classes) : 0;
  jint* p = n ? env->GetIntArrayElements(classes, nullptr) : nullptr;
  const int32_t rc = ks_naive_bayes_fit(ctx, features, sparse, reinterpret_cast<const int32_t*>(p), n, numClasses, lambda, &h);
  if (p) env->ReleaseIntArrayElements(classes, p, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
// ---- the text front end (DESIGN.md section 23): documents and tokens arrive as UTF-8 bytes with int64 offsets; every handle is a
// text object released by textDestroy, except the sparse matrices that sparseFeaturesApply / hashingTf return
struct Bytes {  // borrowed view of a jbyteArray
  JNIEnv* env;
  jbyteArray arr;
  jbyte* p = nullptr;
  jsize n = 0;
  Bytes(JNIEnv* e, jbyteArray a) : env(e), arr(a) {
    if (arr) {
      n = env->GetArrayLength(arr);
      if (n) p = env->GetByteArrayElements(arr, nullptr);
    }
  }
  ~Bytes() {
    if (p) env->ReleaseByteArrayElements(arr, p, JNI_ABORT);
  }
  const uint8_t* data() const { return reinterpret_cast<const uint8_t*>(p); }
};
struct Ints {  // borrowed view of a jintArray
  JNIEnv* env;
  jintArray arr;
  jint* p = nullptr;
  jsize n = 0;
  Ints(JNIEnv* e, jintArray a) : env(e), arr(a) {
    if (arr) {
      n = env->GetArrayLength(arr);
      if (n) p = env->GetIntArrayElements(arr, nullptr);
    }
  }
  ~Ints() {
    if (p) env->ReleaseIntArrayElements(arr, p, JNI_ABORT);
  }
  const int32_t* data() const { return reinterpret_cast<const int32_t*>(p); }
};
struct Doubles {  // borrowed view of a jdoubleArray
  JNIEnv* env;
  jdoubleArray arr;
  jdouble* p = nullptr;
  jsize n = 0;
  Doubles(JNIEnv* e, jdoubleArray a) : env(e), arr(a) {
    if (arr) {
      n = env->GetArrayLength(arr);
      if (n) p = env->GetDoubleArrayElements(arr, nullptr);
    }
  }
  ~Doubles() {
    if (p) env->ReleaseDoubleArrayElements(arr, p, JNI_ABORT);
  }
};

JFN(jlong, textFromHost)(JNIEnv* env, jobject, jlong ctx, jbyteArray bytes, jlongArray docOffsets) {
  int64_t h = 0;
  Bytes b(env, bytes);
  LongArray off(env, docOffsets);
  const int32_t rc = ks_text_from_host(ctx, b.data(), b.n, off.data(), off.n > 0 ? off.n - 1 : 0, &h);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, textTransform)(JNIEnv* env, jobject, jlong ctx, jlong text, jint flags) {
  int64_t h = 0;
  return ok(env, ctx, ks_text_transform(ctx, text, flags, &h)) ? h : 0;
}
JFN(jlong, textTokenize)(JNIEnv* env, jobject, jlong ctx, jlong text) {
  int64_t h = 0;
  return ok(env, ctx, ks_text_tokenize(ctx, text, &h)) ? h : 0;
}
JFN(jlong, tokensFromHost)(JNIEnv* env, jobject, jlong ctx, jbyteArray bytes, jlongArray tokenOffsets, jlongArray docOffsets) {
  int64_t h = 0;
  Bytes b(env, bytes);
  LongArray toff(env, tokenOffsets), doff(env, docOffsets);
  const int32_t rc = ks_tokens_from_host(ctx, b.data(), b.n, toff.data(), toff.n > 0 ? toff.n - 1 : 0, doff.data(), doff.n > 0 ? doff.n - 1 : 0, &h);
  return ok(env, ctx, rc) ? h : 0;
}
// returns (term-frequency handle, largest count)
JFN(jlongArray, termFrequency)(JNIEnv* env, jobject, jlong ctx, jlong tokens, jint minOrder, jint maxOrder) {
  int64_t h = 0, mc = 0;
  if (!ok(env, ctx, ks_term_frequency(ctx, tokens, minOrder, maxOrder, &h, &mc))) return nullptr;
  jlongArray out = env->NewLongArray(2);
  if (!out) return nullptr;
  const jlong v[2] = {h, mc};
  env->SetLongArrayRegion(out, 0, 2, v);
  return out;
}
JFN(void, tfSetWeights)(JNIEnv* env, jobject, jlong ctx, jlong tf, jdoubleArray table) {
  Doubles t(env, table);
  ok(env, ctx, ks_tf_set_weights(ctx, tf, t.p, t.n));
}
JFN(jlong, tfFromHost)(JNIEnv* env, jobject, jlong ctx, jlong tokens, jlongArray termFirst, jintArray termOrder, jdoubleArray values,
                       jlongArray docOffsets) {
  int64_t h = 0;
  LongArray first(env, termFirst), doff(env, docOffsets);
  Ints order(env, termOrder);
  Doubles v(env, values);
  const int32_t rc = ks_tf_from_host(ctx, tokens, first.data(), order.data(), v.p, first.n, doff.data(), doff.n > 0 ? doff.n - 1 : 0, &h);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, sparseFeaturesFit)(JNIEnv* env, jobject, jlong ctx, jlong tf, jlong numFeatures) {
  int64_t h = 0;
  return ok(env, ctx, ks_sparse_features_fit(ctx, tf, numFeatures, &h)) ? h : 0;
}
JFN(jlong, sparseFeaturesFromHost)(JNIEnv* env, jobject, jlong ctx, jlong tokens, jlongArray termFirst, jintArray termOrder) {
  int64_t h = 0;
  LongArray first(env, termFirst);
  Ints order(env, termOrder);
  return ok(env, ctx, ks_sparse_features_from_host(ctx, tokens, first.data(), order.data(), first.n, &h)) ? h : 0;
}
JFN(jlong, sparseFeaturesApply)(JNIEnv* env, jobject, jlong ctx, jlong space, jlong tf) {
  int64_t h = 0;
  return ok(env, ctx, ks_sparse_features_apply(ctx, space, tf, &h)) ? h : 0;
}
JFN(jlong, hashingTf)(JNIEnv* env, jobject, jlong ctx, jlong tokens, jint minOrder, jint maxOrder, jlong numFeatures) {
  int64_t h = 0;
  return ok(env, ctx, ks_hashing_tf(ctx, tokens, minOrder, maxOrder, numFeatures, &h)) ? h : 0;
}
// a text object's array `which` (KS_TEXT_*) as bytes, ints, longs or doubles, whichever its element type is
static jsize text_array_size(JNIEnv* env, jlong ctx, jlong obj, jint which, bool* good) {
  int64_t n = 0;
  *good = ok(env, ctx, ks_text_array_size(ctx, obj, which, &n));
  return static_cast<jsize>(n);
}
JFN(jbyteArray, textArrayBytes)(JNIEnv* env, jobject, jlong ctx, jlong obj, jint which) {
  bool good;
  const jsize n = text_array_size(env, ctx, obj, which, &good);
  if (!good) return nullptr;
  std::vector<jbyte> v(n);
  if (!ok(env, ctx, ks_text_array(ctx, obj, which, v.data(), n))) return nullptr;
  jbyteArray out = env->NewByteArray(n);
  if (out) env->SetByteArrayRegion(out, 0, n, v.data());
  return out;
}
JFN(jintArray, textArrayInts)(JNIEnv* env, jobject, jlong ctx, jlong obj, jint which) {
  bool good;
  const jsize n = text_array_size(env, ctx, obj, which, &good);
  if (!good) return nullptr;
  std::vector<jint> v(n);
  if (!ok(env, ctx, ks_text_array(ctx, obj, which, v.data(), n))) return nullptr;
  jintArray out = env->NewIntArray(n);
  if (out) env->SetIntArrayRegion(out, 0, n, v.data());
  return out;
}
JFN(jlongArray, textArrayLongs)(JNIEnv* env, jobject, jlong ctx, jlong obj, jint which) {
  bool good;
  const jsize n = text_array_size(env, ctx, obj, which, &good);
  if (!good) return nullptr;
  std::vector<jlong> v(n);
  if (!ok(env, ctx, ks_text_array(ctx, obj, which, v.data(), n))) return nullptr;
  jlongArray out = env->NewLongArray(n);
  if (out) env->SetLongArrayRegion(out, 0, n, v.data());
  return out;
}
JFN(jdoubleArray, textArrayDoubles)(JNIEnv* env, jobject, jlong ctx, jlong obj, jint which) {
  bool good;
  const jsize n = text_array_size(env, ctx, obj, which, &good);
  if (!good) return nullptr;
  std::vector<jdouble> v(n);
  if (!ok(env, ctx, ks_text_array(ctx, obj, which, v.data(), n))) return nullptr;
  jdoubleArray out = env->NewDoubleArray(n);
  if (out) env->SetDoubleArrayRegion(out, 0, n, v.data());
  return out;
}
JFN(void, textDestroy)(JNIEnv*, jobject, jlong ctx, jlong obj) { ks_text_destroy(ctx, obj); }
// a sparse matrix as (indptr, indices, values); the Scala side turns row r into a SparseVector
JFN(jobjectArray, sparseToHostCsr)(JNIEnv* env, jobject, jlong ctx, jlong s) {  // [long[] indptr, int[] indices, double[] values]
  int64_t rows = 0, cols = 0, nnz = 0;
  if (!ok(env, ctx, ks_sparse_shape(ctx, s, &rows, &cols, &nnz))) return nullptr;
  std::vector<int64_t> ip(rows + 1);
  std::vector<int32_t> ix(nnz);
  std::vector<double> v(nnz);
  if (!ok(env, ctx, ks_sparse_to_host_csr(ctx, s, ip.data(), ix.data(), v.data()))) return nullptr;
  jclass objc = env->FindClass("java/lang/Object");
  if (!objc) return nullptr;
  jobjectArray out = env->NewObjectArray(3, objc, nullptr);
  jlongArray a = env->NewLongArray(static_cast<jsize>(rows + 1));
  jintArray b = env->NewIntArray(static_cast<jsize>(nnz));
  jdoubleArray d = env->NewDoubleArray(static_cast<jsize>(nnz));
  if (!out || !a || !b || !d) return nullptr;
  env->SetLongArrayRegion(a, 0, static_cast<jsize>(rows + 1), reinterpret_cast<const jlong*>(ip.data()));
  env->SetIntArrayRegion(b, 0, static_cast<jsize>(nnz), ix.data());
  env->SetDoubleArrayRegion(d, 0, static_cast<jsize>(nnz), v.data());
  env->SetObjectArrayElement(out, 0, a);
  env->SetObjectArrayElement(out, 1, b);
  env->SetObjectArrayElement(out, 2, d);
  return out;
}
JFN(jlong, linearMapFit)(JNIEnv* env, jobject, jlong ctx, jlong features, jlong labels, jboolean hasLambda, jdouble lambda) {
  int64_t h = 0;
  return ok(env, ctx, ks_linear_map_fit(ctx, features, labels, hasLambda ? 1 : 0, lambda, &h)) ? h : 0;
}

// ---- PCA / ZCA whitening / approximate PCA (models are ordinary model handles)
JFN(jlong, pcaFit)(JNIEnv* env, jobject, jlong ctx, jlong x, jint dims) {
  int64_t h = 0;
  return ok(env, ctx, ks_pca_fit(ctx, x, dims, &h)) ? h : 0;
}
JFN(jlong, zcaFit)(JNIEnv* env, jobject, jlong ctx, jlong x, jdouble eps) {
  int64_t h = 0;
  return ok(env, ctx, ks_zca_fit(ctx, x, eps, &h)) ? h : 0;
}
// omega: the d x l test matrix as DenseMatrix.data (column-major)
JFN(jlong, approxRange)(JNIEnv* env, jobject, jlong ctx, jlong x, jdoubleArray omega, jint l, jint q) {
  int64_t h = 0;
  jdouble* om = omega ? env->GetDoubleArrayElements(omega, nullptr) : nullptr;
  const int32_t rc = ks_approx_range(ctx, x, om, l, q, &h);
  if (om) env->ReleaseDoubleArrayElements(omega, om, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, approxPcaFit)(JNIEnv* env, jobject, jlong ctx, jlong x, jdoubleArray omega, jint dims, jint q, jint p) {
  int64_t h = 0;
  jdouble* om = omega ? env->GetDoubleArrayElements(omega, nullptr) : nullptr;
  const int32_t rc = ks_approx_pca_fit(ctx, x, om, dims, q, p, &h);
  if (om) env->ReleaseDoubleArrayElements(omega, om, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}

// ---- LCS descriptors, GMM posteriors, Fisher vectors, row normalisation (not collective)
JFN(jlong, lcsExtract)(JNIEnv* env, jobject, jlong ctx, jlong images, jint xDim, jint yDim, jint channels, jint stride, jint strideStart,
                       jint subPatchSize) {
  int64_t h = 0;
  return ok(env, ctx, ks_lcs_extract(ctx, images, xDim, yDim, channels, stride, strideStart, subPatchSize, &h)) ? h : 0;
}
// means / variances: D x K DenseMatrix.data (column-major)
JFN(jlong, gmmCreate)(JNIEnv* env, jobject, jlong ctx, jdoubleArray means, jdoubleArray variances, jdoubleArray weights, jlong dim, jlong k,
                      jdouble weightThreshold) {
  int64_t h = 0;
  jdouble* mu = env->GetDoubleArrayElements(means, nullptr);
  jdouble* var = env->GetDoubleArrayElements(variances, nullptr);
  jdouble* w = env->GetDoubleArrayElements(weights, nullptr);
  const int32_t rc = (mu && var && w) ? ks_gmm_create(ctx, mu, var, w, dim, k, weightThreshold, &h) : KS_ERR_INVALID;
  if (w) env->ReleaseDoubleArrayElements(weights, w, JNI_ABORT);
  if (var) env->ReleaseDoubleArrayElements(variances, var, JNI_ABORT);
  if (mu) env->ReleaseDoubleArrayElements(means, mu, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(void, gmmDestroy)(JNIEnv* env, jobject, jlong ctx, jlong gmm) { ok(env, ctx, ks_gmm_destroy(ctx, gmm)); }
JFN(jlong, gmmPosteriors)(JNIEnv* env, jobject, jlong ctx, jlong gmm, jlong x) {
  int64_t h = 0;
  return ok(env, ctx, ks_gmm_posteriors(ctx, gmm, x, &h)) ? h : 0;
}
// itemOffsets: nItems + 1 row offsets into the descriptor matrix
JFN(jlong, fisherVectorApply)(JNIEnv* env, jobject, jlong ctx, jlong gmm, jlong descriptors, jlongArray itemOffsets) {
  int64_t h = 0;
  LongArray o(env, itemOffsets);
  const int32_t rc = ks_fisher_vector_apply(ctx, gmm, descriptors, o.data(), o.n - 1, &h);
  return ok(env, ctx, rc) ? h : 0;
}
// ---- GMM EM, k-means++, row gather (not collective; DESIGN.md section 17).  uniforms: the draw rule of the header.
// means / variances out: D x K DenseMatrix.data (column-major); returns the model handle
JFN(jlong, gmmFit)(JNIEnv* env, jobject, jlong ctx, jlong x, jlong k, jint maxIterations, jdouble minClusterSize, jdouble stopTolerance,
                   jdouble weightThreshold, jdouble smallVarianceThreshold, jdouble absoluteVarianceThreshold, jint initialization,
                   jdoubleArray uniforms, jdoubleArray meansOut, jdoubleArray variancesOut, jdoubleArray weightsOut) {
  int64_t h = 0;
  jdouble* u = env->GetDoubleArrayElements(uniforms, nullptr);
  jdouble* mu = env->GetDoubleArrayElements(meansOut, nullptr);
  jdouble* var = env->GetDoubleArrayElements(variancesOut, nullptr);
  jdouble* w = env->GetDoubleArrayElements(weightsOut, nullptr);
  const int32_t rc = (u && mu && var && w) ? ks_gmm_fit(ctx, x, k, maxIterations, minClusterSize, stopTolerance, weightThreshold,
                                                        smallVarianceThreshold, absoluteVarianceThreshold, initialization, u, &h, mu,
                                                        var, w, nullptr)
                                           : KS_ERR_INVALID;
  if (w) env->ReleaseDoubleArrayElements(weightsOut, w, 0);
  if (var) env->ReleaseDoubleArrayElements(variancesOut, var, 0);
  if (mu) env->ReleaseDoubleArrayElements(meansOut, mu, 0);
  if (u) env->ReleaseDoubleArrayElements(uniforms, u, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
// meansOut: numMeans x dim row-major; returns the number of Lloyd passes
JFN(jint, kmeansFit)(JNIEnv* env, jobject, jlong ctx, jlong x, jlong numMeans, jint maxIterations, jdouble stopTolerance,
                     jdoubleArray uniforms, jdoubleArray meansOut) {
  int32_t it = 0;
  jdouble* u = env->GetDoubleArrayElements(uniforms, nullptr);
  jdouble* mu = env->GetDoubleArrayElements(meansOut, nullptr);
  const int32_t rc = (u && mu) ? ks_kmeans_fit(ctx, x, numMeans, maxIterations, stopTolerance, u, mu, nullptr, &it) : KS_ERR_INVALID;
  if (mu) env->ReleaseDoubleArrayElements(meansOut, mu, 0);
  if (u) env->ReleaseDoubleArrayElements(uniforms, u, JNI_ABORT);
  return ok(env, ctx, rc) ? it : 0;
}
JFN(jlong, kmeansAssign)(JNIEnv* env, jobject, jlong ctx, jlong x, jdoubleArray meansRowMajor, jlong numMeans, jlong dim) {
  int64_t h = 0;
  jdouble* mu = env->GetDoubleArrayElements(meansRowMajor, nullptr);
  const int32_t rc = mu ? ks_kmeans_assign(ctx, x, mu, numMeans, dim, &h) : KS_ERR_INVALID;
  if (mu) env->ReleaseDoubleArrayElements(meansRowMajor, mu, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, matrixGatherRows)(JNIEnv* env, jobject, jlong ctx, jlong m, jlongArray rows) {
  int64_t h = 0;
  LongArray r(env, rows);
  return ok(env, ctx, ks_matrix_gather_rows(ctx, m, r.data(), r.n, &h)) ? h : 0;
}
// ---- PixelScaler, GrayScaler, dense SIFT (not collective)
JFN(jlong, imagePixelScale)(JNIEnv* env, jobject, jlong ctx, jlong images) {
  int64_t h = 0;
  return ok(env, ctx, ks_image_pixel_scale(ctx, images, &h)) ? h : 0;
}
JFN(jlong, imageGrayscale)(JNIEnv* env, jobject, jlong ctx, jlong images, jint xDim, jint yDim, jint channels, jint pixelScale) {
  int64_t h = 0;
  return ok(env, ctx, ks_image_grayscale(ctx, images, xDim, yDim, channels, pixelScale, &h)) ? h : 0;
}
JFN(jlong, siftExtract)(JNIEnv* env, jobject, jlong ctx, jlong grayImages, jint xDim, jint yDim, jint step, jint bin, jint scales,
                        jint scaleStep) {
  int64_t h = 0;
  return ok(env, ctx, ks_sift_extract(ctx, grayImages, xDim, yDim, step, bin, scales, scaleStep, &h)) ? h : 0;
}
// per-scale keypoint counts (host only); null when the arguments are rejected
JFN(jlongArray, siftKeypoints)(JNIEnv* env, jobject, jint xDim, jint yDim, jint step, jint bin, jint scales, jint scaleStep) {
  if (scales < 1) return nullptr;
  std::vector<int64_t> counts(static_cast<size_t>(scales));
  if (ks_sift_keypoints(xDim, yDim, step, bin, scales, scaleStep, counts.data()) != KS_OK) return nullptr;
  jlongArray out = env->NewLongArray(scales);
  if (out) env->SetLongArrayRegion(out, 0, scales, reinterpret_cast<const jlong*>(counts.data()));
  return out;
}
// ---- HOG and DAISY (not collective)
JFN(jlong, hogExtract)(JNIEnv* env, jobject, jlong ctx, jlong images, jint xDim, jint yDim, jint channels, jint pixelScale, jint bin) {
  int64_t h = 0;
  return ok(env, ctx, ks_hog_extract(ctx, images, xDim, yDim, channels, pixelScale, bin, &h)) ? h : 0;
}
JFN(jlong, daisyExtract)(JNIEnv* env, jobject, jlong ctx, jlong grayImages, jint xDim, jint yDim, jint daisyT, jint daisyQ, jint daisyR,
                         jint daisyH, jint pixelBorder, jint stride) {
  int64_t h = 0;
  return ok(env, ctx, ks_daisy_extract(ctx, grayImages, xDim, yDim, daisyT, daisyQ, daisyR, daisyH, pixelBorder, stride, &h)) ? h : 0;
}
JFN(jlong, matrixNormalizeRows)(JNIEnv* env, jobject, jlong ctx, jlong m) {
  int64_t h = 0;
  return ok(env, ctx, ks_matrix_normalize_rows(ctx, m, &h)) ? h : 0;
}
// op 2 of ks_matrix_map: sign(x) sqrt(|x|)
JFN(jlong, matrixSignedSqrt)(JNIEnv* env, jobject, jlong ctx, jlong m) {
  int64_t h = 0;
  return ok(env, ctx, ks_matrix_map(ctx, m, 2, nullptr, 0.0, 0.0, &h)) ? h : 0;
}

// ---- models
JFN(jlong, modelFromHost)(JNIEnv* env, jobject, jlong ctx, jobjectArray xs, jint blockSize, jlong k, jdoubleArray bOrNull,
                          jobjectArray meansOrNull) {
  const jsize nb = env->GetArrayLength(xs);
  int64_t h = 0;
  // small fixed upper bound keeps this wrapper allocation-free; BlockLinearMapper models have D / blockSize blocks
  enum { kMax = 4096 };
  if (nb <= 0 || nb > kMax) {
    ok(env, ctx, KS_ERR_INVALID);
    return 0;
  }
  static thread_local const double* wp[kMax];
  static thread_local const double* mp[kMax];
  static thread_local int64_t rows[kMax];
  jdoubleArray wa[kMax], ma[kMax];
  jsize got = 0;
  bool fail = false;
  for (; got < nb; ++got) {
    wa[got] = static_cast<jdoubleArray>(env->GetObjectArrayElement(xs, got));
    ma[got] = meansOrNull ? static_cast<jdoubleArray>(env->GetObjectArrayElement(meansOrNull, got)) : nullptr;
    wp[got] = env->GetDoubleArrayElements(wa[got], nullptr);
    mp[got] = ma[got] ? env->GetDoubleArrayElements(ma[got], nullptr) : nullptr;
    rows[got] = env->GetArrayLength(wa[got]) / k;
    if (!wp[got] || (ma[got] && !mp[got])) {
      fail = true;
      ++got;
      break;
    }
  }
  jdouble* b = (!fail && bOrNull) ? env->GetDoubleArrayElements(bOrNull, nullptr) : nullptr;
  int32_t rc = KS_ERR_INVALID;
  if (!fail) rc = ks_model_from_host(ctx, wp, rows, nb, k, b, meansOrNull ? mp : nullptr, blockSize, &h);
  if (b) env->ReleaseDoubleArrayElements(bOrNull, b, JNI_ABORT);
  for (jsize j = 0; j < got; ++j) {
    if (wp[j]) env->ReleaseDoubleArrayElements(wa[j], const_cast<jdouble*>(wp[j]), JNI_ABORT);
    if (mp[j]) env->ReleaseDoubleArrayElements(ma[j], const_cast<jdouble*>(mp[j]), JNI_ABORT);
  }
  if (fail) return 0;  // OutOfMemoryError already pending
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jint, modelNumBlocks)(JNIEnv* env, jobject, jlong ctx, jlong model) {
  int32_t nb = 0, bs = 0;
  int64_t k = 0;
  return ok(env, ctx, ks_model_num_blocks(ctx, model, &nb, &k, &bs)) ? nb : 0;
}
// W_j as DenseMatrix.data (column-major rows_j x k), copied out of the pinned host mirror the fit filled while it ran
JFN(jdoubleArray, modelGetBlock)(JNIEnv* env, jobject, jlong ctx, jlong model, jint j) {
  int32_t nb = 0, bs = 0;
  int64_t k = 0, rows = 0;
  const double* w = nullptr;
  if (!ok(env, ctx, ks_model_num_blocks(ctx, model, &nb, &k, &bs))) return nullptr;
  if (!ok(env, ctx, ks_model_block_rows(ctx, model, j, &rows))) return nullptr;
  if (!ok(env, ctx, ks_model_host_view(ctx, model, j, &w, nullptr, nullptr))) return nullptr;
  jdoubleArray out = env->NewDoubleArray(static_cast<jsize>(rows * k));
  if (!out) return nullptr;
  env->SetDoubleArrayRegion(out, 0, static_cast<jsize>(rows * k), w);
  return out;
}
JFN(jdoubleArray, modelGetBlockMean)(JNIEnv* env, jobject, jlong ctx, jlong model, jint j) {
  int64_t rows = 0;
  const double* mu = nullptr;
  if (!ok(env, ctx, ks_model_block_rows(ctx, model, j, &rows))) return nullptr;
  if (!ok(env, ctx, ks_model_host_view(ctx, model, j, nullptr, &mu, nullptr))) return nullptr;
  if (!mu) return nullptr;  // the weighted solver returns no feature scalers
  jdoubleArray out = env->NewDoubleArray(static_cast<jsize>(rows));
  if (!out) return nullptr;
  env->SetDoubleArrayRegion(out, 0, static_cast<jsize>(rows), mu);
  return out;
}
JFN(jdoubleArray, modelGetIntercept)(JNIEnv* env, jobject, jlong ctx, jlong model) {
  int32_t nb = 0, bs = 0;
  int64_t k = 0;
  const double* b = nullptr;
  if (!ok(env, ctx, ks_model_num_blocks(ctx, model, &nb, &k, &bs))) return nullptr;
  if (!ok(env, ctx, ks_model_host_view(ctx, model, 0, nullptr, nullptr, &b))) return nullptr;
  if (!b) return nullptr;
  jdoubleArray out = env->NewDoubleArray(static_cast<jsize>(k));
  if (!out) return nullptr;
  env->SetDoubleArrayRegion(out, 0, static_cast<jsize>(k), b);
  return out;
}
JFN(jlong, modelApply)(JNIEnv* env, jobject, jlong ctx, jlong model, jlong features, jlong xIn, jlongArray rfs) {
  int64_t h = 0;
  LongArray r(env, rfs);
  return ok(env, ctx, ks_model_apply(ctx, model, features, xIn, r.data(), r.n, &h)) ? h : 0;
}
JFN(jintArray, modelApplyArgmax)(JNIEnv* env, jobject, jlong ctx, jlong model, jlong features, jlong xIn, jlongArray rfs, jlong nRows) {
  jintArray out = env->NewIntArray(static_cast<jsize>(nRows));
  if (!out) return nullptr;
  jint* p = env->GetIntArrayElements(out, nullptr);
  if (!p) return nullptr;
  int32_t rc;
  {
    LongArray r(env, rfs);
    rc = ks_model_apply_argmax(ctx, model, features, xIn, r.data(), r.n, reinterpret_cast<int32_t*>(p));
  }
  env->ReleaseIntArrayElements(out, p, 0);
  return ok(env, ctx, rc) ? out : nullptr;
}
JFN(void, modelSave)(JNIEnv* env, jobject, jlong ctx, jlong model, jstring path) {
  const char* s = env->GetStringUTFChars(path, nullptr);
  if (!s) return;
  const int32_t rc = ks_model_save(ctx, model, s);
  env->ReleaseStringUTFChars(path, s);
  ok(env, ctx, rc);
}
JFN(jlong, modelLoad)(JNIEnv* env, jobject, jlong ctx, jstring path) {
  int64_t h = 0;
  const char* s = env->GetStringUTFChars(path, nullptr);
  if (!s) return 0;
  const int32_t rc = ks_model_load(ctx, s, &h);
  env->ReleaseStringUTFChars(path, s);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(void, modelDestroy)(JNIEnv*, jobject, jlong ctx, jlong model) { ks_model_destroy(ctx, model); }

// ---- Gaussian-kernel ridge regression
JFN(jlong, gaussianKernelCreate)(JNIEnv* env, jobject, jlong ctx, jlong xTrain, jdouble gamma) {
  int64_t h = 0;
  return ok(env, ctx, ks_gaussian_kernel_create(ctx, xTrain, gamma, &h)) ? h : 0;
}
JFN(jlong, gaussianKernelBlock)(JNIEnv* env, jobject, jlong ctx, jlong kernel, jlong x, jlong col0, jlong cols) {
  int64_t h = 0;
  return ok(env, ctx, ks_gaussian_kernel_block(ctx, kernel, x, col0, cols, &h)) ? h : 0;
}
JFN(jlong, gaussianKernelNumTrain)(JNIEnv* env, jobject, jlong ctx, jlong kernel) {
  int64_t n = 0;
  return ok(env, ctx, ks_gaussian_kernel_shape(ctx, kernel, &n, nullptr)) ? n : 0;
}
JFN(void, gaussianKernelDestroy)(JNIEnv*, jobject, jlong ctx, jlong kernel) { ks_gaussian_kernel_destroy(ctx, kernel); }
JFN(jlong, krrFit)(JNIEnv* env, jobject, jlong ctx, jlong kernel, jlong labels, jdouble lambda, jint blockSize, jint numEpochs,
                   jintArray blockOrderOrNull) {
  int64_t h = 0;
  jint* order = blockOrderOrNull ? env->GetIntArrayElements(blockOrderOrNull, nullptr) : nullptr;
  if (blockOrderOrNull && !order) return 0;  // OutOfMemoryError pending
  const int32_t rc = ks_krr_fit(ctx, kernel, labels, lambda, blockSize, numEpochs, reinterpret_cast<const int32_t*>(order), &h);
  if (order) env->ReleaseIntArrayElements(blockOrderOrNull, order, JNI_ABORT);
  return ok(env, ctx, rc) ? h : 0;
}
JFN(jlong, kernelModelFromHost)(JNIEnv* env, jobject, jlong ctx, jlong kernel, jobjectArray xs, jlong k, jint blockSize) {
  const jsize nb = env->GetArrayLength(xs);
  int64_t h = 0;
  enum { kMax = 1 << 16 };  // KernelBlockLinearMapper models have nTrain / blockSize blocks
  if (nb <= 0 || nb > kMax || k <= 0) {
    ok(env, ctx, KS_ERR_INVALID);
    return 0;
  }
  static thread_local const double* wp[kMax];
  static thread_local int64_t rows[kMax];
  static thread_local jdoubleArray wa[kMax];
  jsize got = 0;
  bool fail = false;
  for (; got < nb; ++got) {
    wa[got] = static_cast<jdoubleArray>(env->GetObjectArrayElement(xs, got));
    wp[got] = env->GetDoubleArrayElements(wa[got], nullptr);
    rows[got] = env->GetArrayLength(wa[got]) / k;
    if (!wp[got]) {
      fail = true;
      ++got;
      break;
    }
  }
  int32_t rc = KS_ERR_INVALID;
  if (!fail) rc = ks_kernel_model_from_host(ctx, kernel, wp, rows, nb, k, blockSize, &h);
  for (jsize j = 0; j < got; ++j)
    if (wp[j]) env->ReleaseDoubleArrayElements(wa[j], const_cast<jdouble*>(wp[j]), JNI_ABORT);
  if (fail) return 0;  // OutOfMemoryError already pending
  return ok(env, ctx, rc) ? h : 0;
}
