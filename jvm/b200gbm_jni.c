/*
 * JNI shim: com.microsoft.ml.lightgbm.lightgbmlibJNI  ->  libb200gbm.so.  This image has no JDK, so the file is type- and link-checked
 * against jvm/stub/jni.h + libb200gbm.so by tests/test_capi_cpu.py::test_jni_shim_compiles_and_links; it has never run inside a JVM.
 * It covers every lightgbmlib.* method and ChunkedArray proxy the reference's Scala code calls (90 natives), and LGBM_BoosterRefit.
 *
 * The reference loads `_lightgbm` and `_lightgbm_swig` from the lightgbmlib jar
 * (lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/LightGBMUtils.scala:38-41) and calls the SWIG-generated
 * class `lightgbmlib`, whose static methods forward to `lightgbmlibJNI` natives taking raw C pointers as jlong
 * (SWIGTYPE_p_* wrappers, read back with SwigPtrWrapper.getCPtrValue, lightgbm/src/main/scala/com/microsoft/lightgbm/SWIG.scala:8-13).
 * Because libb200gbm.so keeps LightGBM's C names and signatures, the shim is mechanical: one native per C function,
 * pointers as jlong, strings via GetStringUTFChars.  Build (on a box with a JDK):
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../include b200gbm_jni.c -L../mmlspark_b200/lib -lb200gbm -o lib_lightgbm_swig.so
 * and ship libb200gbm.so under the resource name lib_lightgbm.so so NativeLoader
 * (core/src/main/scala/com/microsoft/ml/spark/core/env/NativeLoader.java:47-68) needs no change.
 */
#include <jni.h>
#include <stdint.h>
#include <stdlib.h>
#include "b200gbm_c_api.h"

#define JNI_FN(name) JNIEXPORT jint JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_##name
#define P(x) ((void*)(intptr_t)(x))

JNIEXPORT jstring JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_LGBM_1GetLastError(JNIEnv* env, jclass cls) {
  (void)cls;
  return (*env)->NewStringUTF(env, LGBM_GetLastError());
}
JNI_FN(LGBM_1NetworkInit)(JNIEnv* env, jclass cls, jstring machines, jint port, jint timeout, jint n) {
  (void)cls;
  const char* m = (*env)->GetStringUTFChars(env, machines, NULL);
  int rc = LGBM_NetworkInit(m, port, timeout, n);
  (*env)->ReleaseStringUTFChars(env, machines, m);
  return rc;
}
JNI_FN(LGBM_1NetworkFree)(JNIEnv* env, jclass cls) { (void)env; (void)cls; return LGBM_NetworkFree(); }

/* data / out are SWIG pointer wrappers: double_to_voidp_ptr(new_doubleArray(n)), voidpp_handle() */
JNI_FN(LGBM_1DatasetCreateFromMat)(JNIEnv* env, jclass cls, jlong data, jint data_type, jint nrow, jint ncol, jint row_major,
                                    jstring params, jlong reference, jlong out) {
  (void)cls;
  const char* p = (*env)->GetStringUTFChars(env, params, NULL);
  int rc = LGBM_DatasetCreateFromMat(P(data), data_type, nrow, ncol, row_major, p, P(reference), (DatasetHandle*)P(out));
  (*env)->ReleaseStringUTFChars(env, params, p);
  return rc;
}
JNI_FN(LGBM_1DatasetSetField)(JNIEnv* env, jclass cls, jlong h, jstring name, jlong data, jint n, jint type) {
  (void)cls;
  const char* s = (*env)->GetStringUTFChars(env, name, NULL);
  int rc = LGBM_DatasetSetField(P(h), s, P(data), n, type);
  (*env)->ReleaseStringUTFChars(env, name, s);
  return rc;
}
JNI_FN(LGBM_1DatasetGetNumData)(JNIEnv* env, jclass cls, jlong h, jlong out) { (void)env; (void)cls; return LGBM_DatasetGetNumData(P(h), (int*)P(out)); }
JNI_FN(LGBM_1DatasetGetNumFeature)(JNIEnv* env, jclass cls, jlong h, jlong out) { (void)env; (void)cls; return LGBM_DatasetGetNumFeature(P(h), (int*)P(out)); }
JNI_FN(LGBM_1DatasetFree)(JNIEnv* env, jclass cls, jlong h) { (void)env; (void)cls; return LGBM_DatasetFree(P(h)); }

JNI_FN(LGBM_1BoosterCreate)(JNIEnv* env, jclass cls, jlong train, jstring params, jlong out) {
  (void)cls;
  const char* p = (*env)->GetStringUTFChars(env, params, NULL);
  int rc = LGBM_BoosterCreate(P(train), p, (BoosterHandle*)P(out));
  (*env)->ReleaseStringUTFChars(env, params, p);
  return rc;
}
JNI_FN(LGBM_1BoosterLoadModelFromString)(JNIEnv* env, jclass cls, jstring model, jlong out_iters, jlong out) {
  (void)cls;
  const char* m = (*env)->GetStringUTFChars(env, model, NULL);
  int rc = LGBM_BoosterLoadModelFromString(m, (int*)P(out_iters), (BoosterHandle*)P(out));
  (*env)->ReleaseStringUTFChars(env, model, m);
  return rc;
}
JNI_FN(LGBM_1BoosterMerge)(JNIEnv* env, jclass cls, jlong h, jlong other) { (void)env; (void)cls; return LGBM_BoosterMerge(P(h), P(other)); }
JNI_FN(LGBM_1BoosterAddValidData)(JNIEnv* env, jclass cls, jlong h, jlong v) { (void)env; (void)cls; return LGBM_BoosterAddValidData(P(h), P(v)); }
JNI_FN(LGBM_1BoosterFree)(JNIEnv* env, jclass cls, jlong h) { (void)env; (void)cls; return LGBM_BoosterFree(P(h)); }
/* leaf_preds: an int32 array pointer (new_intArray) of nrow x ncol leaf indices */
JNI_FN(LGBM_1BoosterRefit)(JNIEnv* env, jclass cls, jlong h, jlong leaf_preds, jint nrow, jint ncol) {
  (void)env; (void)cls;
  return LGBM_BoosterRefit(P(h), (const int32_t*)P(leaf_preds), nrow, ncol);
}
/* the hot call: one boosting iteration on the GPU */
JNI_FN(LGBM_1BoosterUpdateOneIter)(JNIEnv* env, jclass cls, jlong h, jlong is_finished) {
  (void)env; (void)cls;
  return LGBM_BoosterUpdateOneIter(P(h), (int*)P(is_finished));
}
JNI_FN(LGBM_1BoosterUpdateOneIterCustom)(JNIEnv* env, jclass cls, jlong h, jlong grad, jlong hess, jlong is_finished) {
  (void)env; (void)cls;
  return LGBM_BoosterUpdateOneIterCustom(P(h), (const float*)P(grad), (const float*)P(hess), (int*)P(is_finished));
}
JNI_FN(LGBM_1BoosterResetParameter)(JNIEnv* env, jclass cls, jlong h, jstring params) {
  (void)cls;
  const char* p = (*env)->GetStringUTFChars(env, params, NULL);
  int rc = LGBM_BoosterResetParameter(P(h), p);
  (*env)->ReleaseStringUTFChars(env, params, p);
  return rc;
}
JNI_FN(LGBM_1BoosterGetEval)(JNIEnv* env, jclass cls, jlong h, jint idx, jlong out_len, jlong out) {
  (void)env; (void)cls;
  return LGBM_BoosterGetEval(P(h), idx, (int*)P(out_len), (double*)P(out));
}
/* SWIG convenience: returns the model text, retrying with the reported length (LightGBMBooster.scala:269-274) */
JNIEXPORT jstring JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_LGBM_1BoosterSaveModelToStringSWIG(
    JNIEnv* env, jclass cls, jlong h, jint start_iter, jint num_iter, jint imp_type, jlong buffer_len, jlong out_len) {
  (void)cls;
  int64_t* n = (int64_t*)P(out_len);
  char* buf = (char*)malloc((size_t)buffer_len);
  if (LGBM_BoosterSaveModelToString(P(h), start_iter, num_iter, imp_type, buffer_len, n, buf) != 0) { free(buf); return NULL; }
  if (*n > buffer_len) {
    free(buf);
    buf = (char*)malloc((size_t)*n);
    if (LGBM_BoosterSaveModelToString(P(h), start_iter, num_iter, imp_type, *n, n, buf) != 0) { free(buf); return NULL; }
  }
  jstring s = (*env)->NewStringUTF(env, buf);
  free(buf);
  return s;
}
JNI_FN(LGBM_1BoosterGetPredict)(JNIEnv* env, jclass cls, jlong h, jint idx, jlong out_len, jlong out) {
  (void)env; (void)cls;
  return LGBM_BoosterGetPredict(P(h), idx, (int64_t*)P(out_len), (double*)P(out));
}
JNI_FN(LGBM_1BoosterGetNumClasses)(JNIEnv* env, jclass cls, jlong h, jlong out) { (void)env; (void)cls; return LGBM_BoosterGetNumClasses(P(h), (int*)P(out)); }
JNI_FN(LGBM_1BoosterNumModelPerIteration)(JNIEnv* env, jclass cls, jlong h, jlong out) { (void)env; (void)cls; return LGBM_BoosterNumModelPerIteration(P(h), (int*)P(out)); }
JNI_FN(LGBM_1BoosterNumberOfTotalModel)(JNIEnv* env, jclass cls, jlong h, jlong out) { (void)env; (void)cls; return LGBM_BoosterNumberOfTotalModel(P(h), (int*)P(out)); }
JNI_FN(LGBM_1BoosterGetNumFeature)(JNIEnv* env, jclass cls, jlong h, jlong out) { (void)env; (void)cls; return LGBM_BoosterGetNumFeature(P(h), (int*)P(out)); }
JNI_FN(LGBM_1BoosterFeatureImportance)(JNIEnv* env, jclass cls, jlong h, jint num_iteration, jint type, jlong out) {
  (void)env; (void)cls;
  return LGBM_BoosterFeatureImportance(P(h), num_iteration, type, (double*)P(out));
}
/* LightGBMBooster.scala:471: LGBM_BoosterDumpModelSWIG(handle, start, num, importance_type, buffer_len, out_len*) -> JSON string */
JNIEXPORT jstring JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_LGBM_1BoosterDumpModelSWIG(
    JNIEnv* env, jclass cls, jlong h, jint start_iter, jint num_iter, jint imp_type, jlong buffer_len, jlong out_len) {
  (void)cls;
  int64_t* n = (int64_t*)P(out_len);
  char* buf = (char*)malloc((size_t)(buffer_len > 0 ? buffer_len : 1));
  if (LGBM_BoosterDumpModel(P(h), start_iter, num_iter, imp_type, buffer_len, n, buf) != 0) { free(buf); return NULL; }
  if (*n > buffer_len) {
    free(buf);
    buf = (char*)malloc((size_t)*n);
    if (LGBM_BoosterDumpModel(P(h), start_iter, num_iter, imp_type, *n, n, buf) != 0) { free(buf); return NULL; }
  }
  jstring s = (*env)->NewStringUTF(env, buf);
  free(buf);
  return s;
}

/* ---- dataset entry points with array / string-array arguments --------------------------------------------------- */
/* DatasetAggregator.scala:442-453: indptr / indices / data are SWIG array pointers */
JNI_FN(LGBM_1DatasetCreateFromCSR)(JNIEnv* env, jclass cls, jlong indptr, jint indptr_type, jlong indices, jlong data, jint data_type,
                                    jlong nindptr, jlong nelem, jlong num_col, jstring params, jlong reference, jlong out) {
  (void)cls;
  const char* p = (*env)->GetStringUTFChars(env, params, NULL);
  int rc = LGBM_DatasetCreateFromCSR(P(indptr), indptr_type, (const int32_t*)P(indices), P(data), data_type, nindptr, nelem, num_col, p, P(reference),
                                     (DatasetHandle*)P(out));
  (*env)->ReleaseStringUTFChars(env, params, p);
  return rc;
}
/* LightGBMDataset.scala:22-47: out_ptr is a voidpp (borrowed pointer into the dataset) */
JNI_FN(LGBM_1DatasetGetField)(JNIEnv* env, jclass cls, jlong h, jstring name, jlong out_len, jlong out_ptr, jlong out_type) {
  (void)cls;
  const char* s = (*env)->GetStringUTFChars(env, name, NULL);
  int rc = LGBM_DatasetGetField(P(h), s, (int*)P(out_len), (const void**)P(out_ptr), (int*)P(out_type));
  (*env)->ReleaseStringUTFChars(env, name, s);
  return rc;
}
/* LightGBMDataset.scala:178-186: SWIG maps `const char**` to a Java String[] */
JNI_FN(LGBM_1DatasetSetFeatureNames)(JNIEnv* env, jclass cls, jlong h, jobjectArray names, jint n) {
  (void)cls;
  const char** c = (const char**)malloc(sizeof(char*) * (size_t)(n > 0 ? n : 1));
  jstring* js = (jstring*)malloc(sizeof(jstring) * (size_t)(n > 0 ? n : 1));
  for (jint i = 0; i < n; ++i) { js[i] = (jstring)(*env)->GetObjectArrayElement(env, names, i); c[i] = (*env)->GetStringUTFChars(env, js[i], NULL); }
  int rc = LGBM_DatasetSetFeatureNames(P(h), c, n);
  for (jint i = 0; i < n; ++i) (*env)->ReleaseStringUTFChars(env, js[i], c[i]);
  free(js); free((void*)c);
  return rc;
}

/* ---- per-row prediction: the SWIG convenience overloads take Java arrays first (LightGBMBooster.scala:520-525,539-543) -------- */
JNI_FN(LGBM_1BoosterPredictForMatSingle)(JNIEnv* env, jclass cls, jdoubleArray row, jlong h, jint data_type, jint ncol, jint row_major,
                                          jint predict_type, jint start_iter, jint num_iter, jstring params, jlong out_len, jlong out) {
  (void)cls;
  jdouble* x = (*env)->GetDoubleArrayElements(env, row, NULL);
  const char* p = (*env)->GetStringUTFChars(env, params, NULL);
  int rc = LGBM_BoosterPredictForMatSingle(P(h), x, data_type, ncol, row_major, predict_type, start_iter, num_iter, p, (int64_t*)P(out_len), (double*)P(out));
  (*env)->ReleaseStringUTFChars(env, params, p);
  (*env)->ReleaseDoubleArrayElements(env, row, x, JNI_ABORT);
  return rc;
}
JNI_FN(LGBM_1BoosterPredictForCSRSingle)(JNIEnv* env, jclass cls, jintArray indices, jdoubleArray values, jint nnz, jlong h, jint indptr_type,
                                          jint data_type, jlong nindptr, jlong num_col, jint predict_type, jint start_iter, jint num_iter,
                                          jstring params, jlong out_len, jlong out) {
  (void)cls;
  jint* idx = (*env)->GetIntArrayElements(env, indices, NULL);
  jdouble* val = (*env)->GetDoubleArrayElements(env, values, NULL);
  const char* p = (*env)->GetStringUTFChars(env, params, NULL);
  int32_t indptr[2] = {0, nnz};       /* one row: the overload has no indptr argument */
  int rc = LGBM_BoosterPredictForCSRSingle(P(h), indptr, indptr_type, (const int32_t*)idx, val, data_type, nindptr, nnz, num_col, predict_type, start_iter,
                                           num_iter, p, (int64_t*)P(out_len), (double*)P(out));
  (*env)->ReleaseStringUTFChars(env, params, p);
  (*env)->ReleaseDoubleArrayElements(env, values, val, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, indices, idx, JNI_ABORT);
  return rc;
}

/* ---- metric names: LGBM_BoosterGetEvalNamesSWIG returns a handle to a string array (LightGBMBooster.scala:282-286) ------------- */
typedef struct { int n; char** strs; } StringArray;
JNIEXPORT jlong JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_LGBM_1BoosterGetEvalNamesSWIG(JNIEnv* env, jclass cls, jlong h) {
  (void)env; (void)cls;
  int n = 0;
  if (LGBM_BoosterGetEvalCounts(P(h), &n) != 0) return 0;
  StringArray* a = (StringArray*)malloc(sizeof(StringArray));
  a->n = n; a->strs = (char**)malloc(sizeof(char*) * (size_t)(n > 0 ? n : 1));
  for (int i = 0; i < n; ++i) a->strs[i] = (char*)malloc(256);
  int got = 0; size_t need = 0;
  if (LGBM_BoosterGetEvalNames(P(h), n, &got, 256, &need, a->strs) != 0) {
    for (int i = 0; i < n; ++i) free(a->strs[i]);
    free(a->strs); free(a);
    return 0;                                   /* validateArray turns the null handle into an exception */
  }
  return (jlong)(intptr_t)a;
}
JNIEXPORT jobjectArray JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_StringArrayHandle_1get_1strings(JNIEnv* env, jclass cls, jlong handle) {
  (void)cls;
  StringArray* a = (StringArray*)P(handle);
  jobjectArray out = (*env)->NewObjectArray(env, a->n, (*env)->FindClass(env, "java/lang/String"), NULL);
  for (int i = 0; i < a->n; ++i) (*env)->SetObjectArrayElement(env, out, i, (*env)->NewStringUTF(env, a->strs[i]));
  return out;
}
JNIEXPORT void JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_StringArrayHandle_1free(JNIEnv* env, jclass cls, jlong handle) {
  (void)env; (void)cls;
  StringArray* a = (StringArray*)P(handle);
  for (int i = 0; i < a->n; ++i) free(a->strs[i]);
  free(a->strs); free(a);
}

/* ---- SWIG carray / cpointer helpers (swig/SwigUtils.scala:92-118, LightGBMDataset.scala, LightGBMBooster.scala) ----------------- */
#define JNI_T(ret, name) JNIEXPORT ret JNICALL Java_com_microsoft_ml_lightgbm_lightgbmlibJNI_##name
#define ARRAY_HELPERS(T, jT, Name)                                                                                                           \
  JNI_T(jlong, new_1##Name)(JNIEnv* env, jclass cls, jlong n) { (void)env; (void)cls; return (jlong)(intptr_t)malloc(sizeof(T) * (size_t)(n > 0 ? n : 1)); } \
  JNI_T(void, delete_1##Name)(JNIEnv* env, jclass cls, jlong p) { (void)env; (void)cls; free(P(p)); }                                        \
  JNI_T(jT, Name##_1getitem)(JNIEnv* env, jclass cls, jlong p, jlong i) { (void)env; (void)cls; return (jT)((T*)P(p))[i]; }                  \
  JNI_T(void, Name##_1setitem)(JNIEnv* env, jclass cls, jlong p, jlong i, jT v) { (void)env; (void)cls; ((T*)P(p))[i] = (T)v; }
ARRAY_HELPERS(int, jint, intArray)
ARRAY_HELPERS(float, jfloat, floatArray)
ARRAY_HELPERS(double, jdouble, doubleArray)
#define POINTER_HELPERS(T, jT, Name)                                                                                                         \
  JNI_T(jlong, new_1##Name)(JNIEnv* env, jclass cls) { (void)env; (void)cls; return (jlong)(intptr_t)calloc(1, sizeof(T)); }                  \
  JNI_T(void, delete_1##Name)(JNIEnv* env, jclass cls, jlong p) { (void)env; (void)cls; free(P(p)); }                                        \
  JNI_T(jT, Name##_1value)(JNIEnv* env, jclass cls, jlong p) { (void)env; (void)cls; return (jT)(*(T*)P(p)); }                               \
  JNI_T(void, Name##_1assign)(JNIEnv* env, jclass cls, jlong p, jT v) { (void)env; (void)cls; *(T*)P(p) = (T)v; }
POINTER_HELPERS(int, jint, intp)
POINTER_HELPERS(int32_t, jint, int32_1tp)
POINTER_HELPERS(int64_t, jlong, int64_1tp)
JNI_T(jlong, new_1voidpp)(JNIEnv* env, jclass cls) { (void)env; (void)cls; return (jlong)(intptr_t)calloc(1, sizeof(void*)); }
JNI_T(jlong, voidpp_1handle)(JNIEnv* env, jclass cls) { (void)env; (void)cls; return (jlong)(intptr_t)calloc(1, sizeof(void*)); }
JNI_T(jlong, voidpp_1value)(JNIEnv* env, jclass cls, jlong p) { (void)env; (void)cls; return (jlong)(intptr_t)(*(void**)P(p)); }
JNI_T(jlong, int_1to_1voidp_1ptr)(JNIEnv* env, jclass cls, jlong p) { (void)env; (void)cls; return p; }
JNI_T(jlong, float_1to_1voidp_1ptr)(JNIEnv* env, jclass cls, jlong p) { (void)env; (void)cls; return p; }
JNI_T(jlong, double_1to_1voidp_1ptr)(JNIEnv* env, jclass cls, jlong p) { (void)env; (void)cls; return p; }

/* ---- ChunkedArray<T> proxies (swig/SwigUtils.scala:22-90): the Java proxy passes (cptr, self) ---------------------------------- */
#define CHUNKED(T, jT, Name, Code)                                                                                                           \
  JNI_T(jlong, new_1##Name)(JNIEnv* env, jclass cls, jlong chunk_size) {                                                                     \
    (void)env; (void)cls; ChunkedArrayHandle h = NULL;                                                                                       \
    return B200GBM_ChunkedArrayCreate(Code, chunk_size, &h) == 0 ? (jlong)(intptr_t)h : 0;                                                   \
  }                                                                                                                                          \
  JNI_T(void, delete_1##Name)(JNIEnv* env, jclass cls, jlong h) { (void)env; (void)cls; B200GBM_ChunkedArrayFree(P(h)); }                    \
  JNI_T(void, Name##_1add)(JNIEnv* env, jclass cls, jlong h, jobject self, jT v) { (void)env; (void)cls; (void)self; B200GBM_ChunkedArrayAdd(P(h), (double)v); } \
  JNI_T(jlong, Name##_1get_1add_1count)(JNIEnv* env, jclass cls, jlong h, jobject self) { (void)env; (void)cls; (void)self; return B200GBM_ChunkedArrayGetAddCount(P(h)); } \
  JNI_T(jlong, Name##_1get_1chunks_1count)(JNIEnv* env, jclass cls, jlong h, jobject self) { (void)env; (void)cls; (void)self; return B200GBM_ChunkedArrayGetChunksCount(P(h)); } \
  JNI_T(jlong, Name##_1get_1last_1chunk_1add_1count)(JNIEnv* env, jclass cls, jlong h, jobject self) {                                       \
    (void)env; (void)cls; (void)self; return B200GBM_ChunkedArrayGetLastChunkAddCount(P(h));                                                 \
  }                                                                                                                                          \
  JNI_T(jT, Name##_1getitem)(JNIEnv* env, jclass cls, jlong h, jobject self, jlong chunk, jlong idx, jT on_fail) {                           \
    (void)env; (void)cls; (void)self; return (jT)B200GBM_ChunkedArrayGetItem(P(h), chunk, idx, (double)on_fail);                             \
  }                                                                                                                                          \
  JNI_T(void, Name##_1coalesce_1to)(JNIEnv* env, jclass cls, jlong h, jobject self, jlong out) { (void)env; (void)cls; (void)self; B200GBM_ChunkedArrayCoalesceTo(P(h), P(out)); } \
  JNI_T(void, Name##_1release)(JNIEnv* env, jclass cls, jlong h, jobject self) { (void)env; (void)cls; (void)self; B200GBM_ChunkedArrayRelease(P(h)); }
CHUNKED(float, jfloat, floatChunkedArray, C_API_DTYPE_FLOAT32)
CHUNKED(double, jdouble, doubleChunkedArray, C_API_DTYPE_FLOAT64)
CHUNKED(int32_t, jint, int32ChunkedArray, C_API_DTYPE_INT32)
