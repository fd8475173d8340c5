// Batched prediction on the device of a Booster's model: the flattened forest, the CSR slot table, the TreeSHAP scratch and the chunk
// loop that dense and CSR input share (kernels: predict_kernels.cuh).  Part of engine.cu's translation unit (predictor.cu is included there).
#pragma once
#include "engine.h"
#include "predict_kernels.cuh"

namespace b200gbm {

class Predictor {
 public:
  // model and stream are the booster's, read live; a null stream (prediction-only booster) is acquired here and released by the booster
  Predictor(const HostModel& model, cudaStream_t& stream) : model_(model), stream_(stream) {}
  void Invalidate() { forest_.reset(); }      // leaf values on the device are stale (DART); a new tree count is noticed without this
  // a row-major matrix (host or device pointer); predict_type 0 normal, 1 raw, 2 leaf index, 3 contributions.
  // `es` (PredictEarlyStop) on: normal and raw scores stop early per row (k_predict_raw_es), bit for bit HostModel::PredictRow's.
  // Returns the number of doubles written to `out` (host).  last_ms = kernel time (CUDA events), incl. H2D for host input.
  int64_t PredictMat(const void* data, int data_type, int64_t nrow, int ncol, int predict_type, int start_iteration, int num_iteration,
                     const EarlyStop& es, double* out);
  // the same over a host CSR matrix (indptr_type 2 = int32, 3 = int64; data_type 1 = float64), uploaded in chunks of rows: every output
  // equals PredictMat's on the densified rows.  indptr must start at 0 or above, never decrease and end at most at nelem.
  int64_t PredictCSR(const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr,
                     int64_t nelem, int predict_type, int start_iteration, int num_iteration, const EarlyStop& es, double* out);
  double last_ms = 0.0;

 private:
  // PredictCSR's slots (k_csr_to_slots) for the trees [t0, t1): the U distinct split features in ascending order
  struct SlotBufs { int t0 = 0, t1 = 0, U = 0; DevBuf<int> slot_of_feature, feature_of_slot, split_slot; };
  struct ForestBufs {
    DevBuf<int> tree_offset, leaf_offset, num_leaves, split_feature, decision_type, left_child, right_child, cat_begin, cat_len; DevBuf<double> threshold, leaf_value, node_count, leaf_count, expected; DevBuf<unsigned> cat_words; size_t trees = 0; int max_depth = 0;
    std::unique_ptr<SlotBufs> slots;      // built for the last iteration range PredictCSR was asked for, dropped with the forest
    ForestDev View() const { return ForestDev{tree_offset.p, leaf_offset.p, num_leaves.p, split_feature.p, threshold.p, decision_type.p, left_child.p, right_child.p, leaf_value.p, cat_begin.p, cat_len.p, cat_words.p, node_count.p, leaf_count.p, expected.p}; }
  };
  void UploadForest();
  const SlotBufs& UploadSlots(int t0, int t1);
  template <typename T>
  void LaunchRawEarlyStop(const ForestDev& f, const T* X, int64_t rows, int ncol, int K, int i0, int i1, const EarlyStop& es, double* y);
  template <typename End, typename Stage>
  int64_t Run(int64_t nrow, int64_t chunk, int64_t per_row, int predict_type, int t0, int t1, const EarlyStop& es, double* out, End end,
              Stage stage);

  const HostModel& model_;
  cudaStream_t& stream_;
  std::unique_ptr<ForestBufs> forest_;
};

}  // namespace b200gbm
