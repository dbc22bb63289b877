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
JFN(jlong, linearMapFit)(JNIEnv* env, jobject, jlong ctx, jlong features, jlong labels, jboolean hasLambda, jdouble lambda) {
  int64_t h = 0;
  return ok(env, ctx, ks_linear_map_fit(ctx, features, labels, hasLambda ? 1 : 0, lambda, &h)) ? h : 0;
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
