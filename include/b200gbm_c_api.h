/*
 * b200gbm C ABI — the drop-in boundary of the H100-native LightGBM-on-Spark training path.
 *
 * libb200gbm.so exports the subset of the LightGBM 3.2.x C API that MMLSpark calls through the
 * SWIG-generated `lightgbmlib` bindings (SURVEY.md §8b), with the same names, argument order and
 * error convention (every function returns 0 on success, -1 on failure; the message is read with
 * LGBM_GetLastError()).  Handles are opaque pointers; all input arrays are caller-owned and may be
 * freed as soon as the call returns.  Last-error, CUDA-device and network state are thread-local:
 * one host thread drives one (network, dataset, booster) triple, like one Spark task thread.
 *
 * Citations are into the reference (Azure/mmlspark) lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/ (LGB/).
 * Every `data` pointer may be a host pointer OR a CUDA device pointer (detected at run time).
 * There is no CPU fallback: calls that need the GPU fail with -1 when no CUDA device is present.
 */
#ifndef B200GBM_C_API_H_
#define B200GBM_C_API_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* DatasetHandle;
typedef void* BoosterHandle;

#define C_API_DTYPE_FLOAT32 (0) /* LGB/dataset/LightGBMDataset.scala:35-41 */
#define C_API_DTYPE_FLOAT64 (1)
#define C_API_DTYPE_INT32 (2)
#define C_API_DTYPE_INT64 (3)

#define C_API_PREDICT_NORMAL (0) /* LGB/booster/LightGBMBooster.scala:144-150 */
#define C_API_PREDICT_RAW_SCORE (1)
#define C_API_PREDICT_LEAF_INDEX (2)
#define C_API_PREDICT_CONTRIB (3)

/* ---- error ------------------------------------------------------------------------------ */
/* LGB/LightGBMUtils.scala:22-34 (validate: rc == -1 -> LGBM_GetLastError) */
const char* LGBM_GetLastError(void);

/* ---- network (replaces LightGBM's TCP collectives with NCCL over NVLink) ------------------ */
/* LGB/TrainUtils.scala:279-295: LGBM_NetworkInit(nodes, localListenPort, 120, numNodes).
 * `machines` = "ip:port,ip:port,..."; the rank is the position of the entry whose port equals
 * local_listen_port.  Rank 0 connects to every other rank's listen port, collects each rank's process
 * token and device UUID, and sends back the layout it chose: every rank on its own device -> NCCL (with
 * rank 0's ncclUniqueId), every rank a thread of this process on one device -> the in-process
 * same-device collective (at most 16 ranks).  Any other layout returns -1 on every rank with a message
 * naming the ranks that share a device.  listen_time_out also bounds every same-device collective, and a
 * rank that calls LGBM_NetworkFree early makes the others' collectives fail ("left the network"). */
int LGBM_NetworkInit(const char* machines, int local_listen_port, int listen_time_out, int num_machines);
/* LGB/LightGBMBase.scala:379 */
int LGBM_NetworkFree(void);

/* ---- dataset ---------------------------------------------------------------------------- */
/* LGB/dataset/DatasetAggregator.scala:335-343 (dense) */
int LGBM_DatasetCreateFromMat(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major,
                              const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* LGB/dataset/DatasetAggregator.scala:442-453 (sparse) */
int LGBM_DatasetCreateFromCSR(const void* indptr, int indptr_type, const int32_t* indices, const void* data,
                              int data_type, int64_t nindptr, int64_t nelem, int64_t num_col,
                              const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* [UPSTREAM] LightGBM's LGBM_DatasetCreateFromMats: one dataset from nmat row parts that count as one matrix (part 0's
 * rows, then part 1's, ...).  Each data[i] holds nrow[i] rows and may be a host or a device pointer.  Bins, bundles and
 * mappers, and so every model trained on it, are bit-identical to LGBM_DatasetCreateFromMat on the concatenation; no host
 * copy of the parts is made.  Rejects nmat < 1, a part without rows and null pointers. */
int LGBM_DatasetCreateFromMats(int32_t nmat, const void** data, int data_type, int32_t* nrow, int32_t ncol, int is_row_major,
                               const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* The same for nparts host CSR parts (no upstream equivalent): part i is indptr[i] (nindptr[i] entries, need not start at
 * 0), indices[i] and data[i] (nelem[i] stored values).  Equal to LGBM_DatasetCreateFromCSR on the concatenated rows; every
 * part is checked as LGBM_DatasetCreateFromCSR checks its input. */
int B200GBM_DatasetCreateFromCSRs(int32_t nparts, const void** indptr, int indptr_type, const int32_t** indices,
                                  const void** data, int data_type, const int64_t* nindptr, const int64_t* nelem,
                                  int64_t num_col, const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* LightGBM streaming ingestion (not used by the reference revision; offered as the bulk path of
 * SURVEY.md §8f-1): create from a column-wise sample, then push row blocks (host or device). */
int LGBM_DatasetCreateFromSampledColumn(double** sample_data, int** sample_indices, int32_t ncol,
                                        const int* num_per_col, int32_t num_sample_row, int32_t num_total_row,
                                        const char* parameters, DatasetHandle* out);
int LGBM_DatasetPushRows(DatasetHandle dataset, const void* data, int data_type, int32_t nrow, int32_t ncol,
                         int32_t start_row);
/* LGB/dataset/LightGBMDataset.scala:85-169 ("label"/"weight" f32, "init_score" f64, "group" i32) */
int LGBM_DatasetSetField(DatasetHandle handle, const char* field_name, const void* field_data, int num_element, int type);
/* LGB/dataset/LightGBMDataset.scala:22-47 (borrowed pointer into the dataset) */
int LGBM_DatasetGetField(DatasetHandle handle, const char* field_name, int* out_len, const void** out_ptr, int* out_type);
/* LGB/dataset/LightGBMDataset.scala:52-69 */
int LGBM_DatasetGetNumData(DatasetHandle handle, int* out);
int LGBM_DatasetGetNumFeature(DatasetHandle handle, int* out);
/* LGB/dataset/LightGBMDataset.scala:178-186 */
int LGBM_DatasetSetFeatureNames(DatasetHandle handle, const char** feature_names, int num_feature_names);
/* LGB/dataset/LightGBMDataset.scala:188-191 */
int LGBM_DatasetFree(DatasetHandle handle);

/* ---- booster life cycle ------------------------------------------------------------------ */
/* LGB/booster/LightGBMBooster.scala:230-243 */
int LGBM_BoosterCreate(const DatasetHandle train_data, const char* parameters, BoosterHandle* out);
/* LGB/booster/LightGBMBooster.scala:41-48 */
int LGBM_BoosterLoadModelFromString(const char* model_str, int* out_num_iterations, BoosterHandle* out);
/* LGB/booster/LightGBMBooster.scala:252-256 */
int LGBM_BoosterMerge(BoosterHandle handle, BoosterHandle other_handle);
/* LGB/booster/LightGBMBooster.scala:258-264 */
int LGBM_BoosterAddValidData(BoosterHandle handle, const DatasetHandle valid_data);
/* LGB/booster/LightGBMBooster.scala:152-157 */
int LGBM_BoosterFree(BoosterHandle handle);

/* ---- training (the hot path) ------------------------------------------------------------- */
/* LGB/booster/LightGBMBooster.scala:351-361 — one boosting iteration: gradients -> per-partition
 * histograms (K4) -> NCCL histogram allreduce (C2) -> best-split scan (K5) -> row partition (K7) */
int LGBM_BoosterUpdateOneIter(BoosterHandle handle, int* is_finished);
/* LGB/booster/LightGBMBooster.scala:368-388 (custom objective: grad/hess of length num_data*num_class) */
int LGBM_BoosterUpdateOneIterCustom(BoosterHandle handle, const float* grad, const float* hess, int* is_finished);
/* LGB/booster/LightGBMBooster.scala:315-318 ("learning_rate=<x>") */
int LGBM_BoosterResetParameter(BoosterHandle handle, const char* parameters);

/* LightGBM's LGBM_BoosterRefit (Booster.refit / task=refit): leaf_preds is row-major nrow x ncol, the leaf of training row i in model
 * j (nrow = the training rows, ncol = the models).  Every tree keeps its structure; each leaf value becomes
 * refit_decay_rate * leaf + (1 - refit_decay_rate) * the leaf output of its rows' gradients at the current training scores. */
int LGBM_BoosterRefit(BoosterHandle handle, const int32_t* leaf_preds, int32_t nrow, int32_t ncol);

/* ---- evaluation / introspection ---------------------------------------------------------- */
int LGBM_BoosterGetEvalCounts(BoosterHandle handle, int* out_len);
/* LGB/booster/LightGBMBooster.scala:279-294 (through the SWIG string-array helper) */
int LGBM_BoosterGetEvalNames(BoosterHandle handle, const int len, int* out_len, const size_t buffer_len,
                             size_t* out_buffer_len, char** out_strs);
/* LGB/booster/LightGBMBooster.scala:296-310 */
int LGBM_BoosterGetEval(BoosterHandle handle, int data_idx, int* out_len, double* out_results);
int LGBM_BoosterGetNumPredict(BoosterHandle handle, int data_idx, int64_t* out_len);
/* LGB/booster/LightGBMBooster.scala:327-346 */
int LGBM_BoosterGetPredict(BoosterHandle handle, int data_idx, int64_t* out_len, double* out_result);
/* LGB/booster/LightGBMBooster.scala:159-197 */
int LGBM_BoosterGetNumClasses(BoosterHandle handle, int* out_len);
int LGBM_BoosterNumModelPerIteration(BoosterHandle handle, int* out_tree_per_iteration);
int LGBM_BoosterNumberOfTotalModel(BoosterHandle handle, int* out_models);
int LGBM_BoosterGetNumFeature(BoosterHandle handle, int* out_len);
int LGBM_BoosterGetCurrentIteration(BoosterHandle handle, int* out_iteration);
/* LGB/booster/LightGBMBooster.scala:491-498 */
int LGBM_BoosterFeatureImportance(BoosterHandle handle, int num_iteration, int importance_type, double* out_results);

/* ---- model (de)serialisation ------------------------------------------------------------- */
/* LGB/booster/LightGBMBooster.scala:269-274 (SWIG helper retries with out_len when the buffer is short) */
int LGBM_BoosterSaveModelToString(BoosterHandle handle, int start_iteration, int num_iteration,
                                  int feature_importance_type, int64_t buffer_len, int64_t* out_len, char* out_str);
/* LGB/booster/LightGBMBooster.scala:465-472 */
int LGBM_BoosterDumpModel(BoosterHandle handle, int start_iteration, int num_iteration, int feature_importance_type,
                          int64_t buffer_len, int64_t* out_len, char* out_str);

/* ---- prediction (per-row UDF semantics of the reference; host side) ------------------------ */
/* `parameter` (NULL or "" = no keys): only the prediction early-stopping keys pred_early_stop, pred_early_stop_freq and
 * pred_early_stop_margin are read (see B200GBM_BoosterPredictForMatDeviceWithParameter); every other key is ignored. */
/* LGB/booster/LightGBMBooster.scala:528-545 */
int LGBM_BoosterPredictForMatSingle(BoosterHandle handle, const void* data, int data_type, int ncol, int is_row_major,
                                    int predict_type, int start_iteration, int num_iteration, const char* parameter,
                                    int64_t* out_len, double* out_result);
/* LGB/booster/LightGBMBooster.scala:510-526 */
int LGBM_BoosterPredictForCSRSingle(BoosterHandle handle, const void* indptr, int indptr_type, const int32_t* indices,
                                    const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col,
                                    int predict_type, int start_iteration, int num_iteration, const char* parameter,
                                    int64_t* out_len, double* out_result);
int LGBM_BoosterPredictForMat(BoosterHandle handle, const void* data, int data_type, int32_t nrow, int32_t ncol,
                              int is_row_major, int predict_type, int start_iteration, int num_iteration,
                              const char* parameter, int64_t* out_len, double* out_result);
int LGBM_BoosterCalcNumPredict(BoosterHandle handle, int num_row, int predict_type, int start_iteration,
                               int num_iteration, int64_t* out_len);

/* ---- ChunkedArray<T> (LGB/swig/SwigUtils.scala:22-90): growable chunk list for row streams ---- */
typedef void* ChunkedArrayHandle;
int B200GBM_ChunkedArrayCreate(int data_type, int64_t chunk_size, ChunkedArrayHandle* out);
int B200GBM_ChunkedArrayAdd(ChunkedArrayHandle h, double value);
int B200GBM_ChunkedArrayAddMany(ChunkedArrayHandle h, const void* values, int64_t n);
int64_t B200GBM_ChunkedArrayGetAddCount(ChunkedArrayHandle h);
int64_t B200GBM_ChunkedArrayGetChunksCount(ChunkedArrayHandle h);
int64_t B200GBM_ChunkedArrayGetLastChunkAddCount(ChunkedArrayHandle h);
double B200GBM_ChunkedArrayGetItem(ChunkedArrayHandle h, int64_t chunk, int64_t index, double on_fail);
int B200GBM_ChunkedArrayCoalesceTo(ChunkedArrayHandle h, void* out);
int B200GBM_ChunkedArrayRelease(ChunkedArrayHandle h);
int B200GBM_ChunkedArrayFree(ChunkedArrayHandle h);

/* ---- engine extensions (instrumentation, parity and benchmark support) ----------------------- */
int B200GBM_SetDevice(int ordinal);                 /* thread-local CUDA device of the calling rank-thread */
int B200GBM_GetDevice(int* ordinal);
int B200GBM_DeviceAlloc(size_t bytes, void** out);  /* cudaMalloc / cudaFree on the thread's device */
int B200GBM_DeviceFree(void* ptr);
int B200GBM_HostAllocPinned(size_t bytes, void** out);
int B200GBM_HostFreePinned(void* ptr);
int B200GBM_Memcpy(void* dst, const void* src, size_t bytes);   /* cudaMemcpyDefault + sync */
/* LightGBM's LCG row sampler (the rows that define the bins) */
int B200GBM_SampleIndices(int num_total_row, int sample_cnt, int seed, int* out, int* out_len);
/* counter-based synthetic generators (SURVEY.md §8d): kind 0 = regression, 1 = binary, 2 = graded relevance 0..4 (ranking),
 * 3 = 10 classes with the last ncol/16 columns categorical (log-uniform ids, cardinality 10^3..10^5) and a 70 %-zero first quarter.
 * x(row, col) and label(row) are pure functions of (seed, row, col). */
int B200GBM_SyntheticFill(void* dev_x_f32, void* dev_label_f32, int64_t row_start, int32_t nrow, int32_t ncol,
                          uint64_t seed, int kind);
int B200GBM_SyntheticRows(const int* rows, int32_t nrows, int32_t ncol, uint64_t seed, int kind, double* host_out,
                          float* host_label_out);
/* dataset introspection for the bit-exact bin parity tests */
int B200GBM_DatasetGetBins(DatasetHandle handle, uint8_t* out_row_major);          /* [num_data][num_feature] */
int B200GBM_DatasetGetBins16(DatasetHandle handle, uint16_t* out_row_major);       /* same, uint16: datasets with features of more than 256 bins */
int B200GBM_DatasetGetBinToCat(DatasetHandle handle, int feature, int* out, int* out_len);   /* categorical feature: bin -> category value (out: >= num_bin ints) */
/* bins of the selected rows only, gathered on the device: out [nrows][num_feature] uint16 (trivial features 0).  Lets a test or
 * bench.py check rows of a dataset far too large to download (the 100M x 512 benchmark matrix) against host-side binning. */
int B200GBM_DatasetGetBinsRows(DatasetHandle handle, const int32_t* rows, int32_t nrows, uint16_t* out);
/* storage layout of the uint8 bins: out_num_columns = storage columns (feature bundles + plain features + wide features), out_column_of
 * [num_feature] = the column of each feature, -1 if unused.  Features of one exclusive feature bundle share a column. */
int B200GBM_DatasetGetBundles(DatasetHandle handle, int* out_num_columns, int* out_column_of);
/* {min, max} of the sampled values of a feature (the feature_infos entry of the model text) */
int B200GBM_DatasetGetFeatureRange(DatasetHandle handle, int feature, double* out2);
int B200GBM_DatasetGetFeatureInfo(DatasetHandle handle, int feature, int* out5);   /* num_bin, missing, default_bin, most_freq_bin, trivial */
int B200GBM_DatasetGetUpperBounds(DatasetHandle handle, int feature, double* out, int* out_len);
int B200GBM_DatasetGetIngestMs(DatasetHandle handle, double* out_ms);
/* kernel-level entry: fixed-point histogram (K4) of the given rows on the dataset's bins, returned as
 * fp64 [num_feature][256][2]; grad/hess/idx are host arrays; idx == NULL means rows 0..cnt-1 */
int B200GBM_DatasetHistogram(DatasetHandle handle, const float* grad, const float* hess, const int32_t* idx,
                             int32_t cnt, double* out);
/* kernel-level entry of quantised training (use_quantized_grad): the training path's discretisation of grad/hess into
 * num_grad_quant_bins levels (stochastic rounding keyed by seed = data_random_seed and tree_index) and its packed K4 histogram of the
 * given rows.  out_q [num_data][2] the levels (q_g, q_h), out_scale2 {s_g, s_h}, out_hist [num_feature][256][2] the int64 sums of q.
 * hess == NULL: constant hessians (q_h = 1 per row, s_h = 1); idx == NULL means rows 0..cnt-1 */
int B200GBM_DatasetQuantizedHistogram(DatasetHandle handle, const float* grad, const float* hess, const int32_t* idx, int32_t cnt,
                                      int num_grad_quant_bins, int stochastic_rounding, int seed, int tree_index, int32_t* out_q,
                                      double* out_scale2, int64_t* out_hist);
/* kernel-level entry: the objective's gradients and hessians (K1/K2) at the booster's current training scores, class-major [K][n]
 * host arrays; classes the objective does not train read back as 0.  Training state and the model are not changed. */
int B200GBM_BoosterGetGradients(BoosterHandle handle, float* grad, float* hess);
/* the ranking objectives' position factors (a training set with the "position" field, lambdarank or rank_xendcg): out_len = the number
 * of distinct position values over every rank's training rows; when buffer_len >= out_len, out_ids [out_len] gets those values in
 * ascending order and out_factors [out_len] the factor of each.  A booster with no position field (or another objective, or loaded from
 * a model string) gives out_len = 0.  The factors are training state: model text and predictions do not contain them. */
int B200GBM_BoosterGetPositionBias(BoosterHandle handle, int64_t buffer_len, int* out_len, int32_t* out_ids, double* out_factors);
/* the last LGBM_BoosterRefit: out = {staging ms, per-tree work ms (host clock, each ending in a device sync), batches of models,
 * row blocks staged} */
int B200GBM_BoosterGetRefitTiming(BoosterHandle handle, double* out4);
/* timing of the engine stream, CUDA events: out = {hist_ms, total_ms, hist_rows, hist_launches, launches, iterations} */
int B200GBM_BoosterSetProfile(BoosterHandle handle, int profile_hist);
int B200GBM_BoosterGetTiming(BoosterHandle handle, double* out6, int reset);
int B200GBM_BoosterGetScores(BoosterHandle handle, int data_idx, double* out);    /* raw scores, class-major */
/* batched GPU prediction (SURVEY §8f-2): row-major matrix on the host or the device, predict_type NORMAL / RAW_SCORE / LEAF_INDEX /
 * CONTRIB (TreeSHAP, [nrow][num_class][num_feature+1]); values equal LGBM_BoosterPredictForMatSingle row by row (raw scores and leaf
 * indices bit for bit, contributions to 1e-12); out_result is a host buffer sized by LGBM_BoosterCalcNumPredict; elapsed_ms (may be
 * NULL) = CUDA-event time.  Replaces the per-row UDF calls of LightGBMBooster.scala:390-423,528-545 for whole partitions. */
int B200GBM_BoosterPredictForMatDevice(BoosterHandle handle, const void* data, int data_type, int64_t nrow, int32_t ncol, int predict_type,
                                       int start_iteration, int num_iteration, int64_t* out_len, double* out_result, double* elapsed_ms);
/* B200GBM_BoosterPredictForMatDevice with the predict call's parameter string, in the position LightGBM's predict functions take it
 * (NULL or "" = no keys, the same outputs bit for bit).  The keys read are pred_early_stop, pred_early_stop_freq (default 10) and
 * pred_early_stop_margin (default 10.0), as LGBM_BoosterPredictForMat* read them: for a binary, multiclass, multiclassova, lambdarank or
 * rank_xendcg model and a NORMAL or RAW_SCORE prediction, a row walks no more trees once, after a multiple of freq iterations, its
 * margin (2|s| for one score, the largest minus the second largest score otherwise) exceeds the margin.  Outputs equal the single-row
 * entries' with the same string bit for bit.  freq <= 0 or a margin < 0 (or NaN) fails the call when early stopping applies. */
int B200GBM_BoosterPredictForMatDeviceWithParameter(BoosterHandle handle, const void* data, int data_type, int64_t nrow, int32_t ncol,
                                                    int predict_type, int start_iteration, int num_iteration, const char* parameter,
                                                    int64_t* out_len, double* out_result, double* elapsed_ms);
/* batched GPU prediction of a host CSR matrix (indptr INT32 or INT64, data FLOAT64), arguments of LGBM_BoosterPredictForCSRSingle plus
 * elapsed_ms.  Every output equals B200GBM_BoosterPredictForMatDevice on the densified rows bit for bit (a missing entry is 0, of
 * repeated indices the last wins, indices outside the model's features are ignored), and so LGBM_BoosterPredictForCSRSingle on the row:
 * bit for bit, contributions to 1e-12.  Contributions keep the dense layout [nrow][num_class][num_feature+1].  Only the features the
 * trees split on are built on the device, so a row costs O(its nonzeros + the split features) however wide num_col is.  Unlike the
 * single-row entry, a bad indptr (decreasing, negative, or past nelem) is an error. */
int B200GBM_BoosterPredictForCSRDevice(BoosterHandle handle, const void* indptr, int indptr_type, const int32_t* indices, const void* data,
                                       int data_type, int64_t nindptr, int64_t nelem, int64_t num_col, int predict_type, int start_iteration,
                                       int num_iteration, int64_t* out_len, double* out_result, double* elapsed_ms);
/* B200GBM_BoosterPredictForCSRDevice with the predict call's parameter string, read as by B200GBM_BoosterPredictForMatDeviceWithParameter */
int B200GBM_BoosterPredictForCSRDeviceWithParameter(BoosterHandle handle, const void* indptr, int indptr_type, const int32_t* indices,
                                                    const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col,
                                                    int predict_type, int start_iteration, int num_iteration, const char* parameter,
                                                    int64_t* out_len, double* out_result, double* elapsed_ms);
/* out = {num_machines, rank, histogram reduce mode (0 = ncclAllReduce, 3 = same-device all-reduce: every rank a thread of this process
 * on this device), constant_hessian} */
int B200GBM_BoosterGetInfo(BoosterHandle handle, int* out4);
/* out = {bytes of the optional column-major copy of the training bins kept for the partition kernel (0 = not kept: it is set up before the
 * first tree only within a reserve of device memory, B200GBM_COLUMN_COPY=0 disables it; when the full copy does not fit, the bytes of
 * the column cache's slot pool), free device memory in bytes} */
int B200GBM_BoosterGetMemoryInfo(BoosterHandle handle, int64_t* out2);
/* out = {slots of the column cache (0 = no cache: full copy or none), slots in use, columns built into slots so far, evictions so far} */
int B200GBM_BoosterGetColumnCacheInfo(BoosterHandle handle, int64_t* out4);
/* out = {histogram bytes all-reduced by this rank (data-parallel: the whole histogram slot per split round; voting-parallel: the packed
 * buffer of 2 * top_k voted storage columns and the two leaves' totals), vote record bytes all-gathered (all ranks' records, voting only),
 * split rounds enqueued (num_leaves - 1 per tree, also when a tree stops early)}, all since the booster was created; 0 bytes on one rank */
int B200GBM_BoosterGetCommInfo(BoosterHandle handle, int64_t* out3);

#ifdef __cplusplus
}
#endif
#endif /* B200GBM_C_API_H_ */
