// Predictor (predictor.h).  Included by engine.cu: one translation unit with the kernels it launches.
#include "predictor.h"

namespace b200gbm {

// bounds of one chunk: bytes of input rows staged on the device, bytes of output (contributions are wide), nonzeros of CSR input
constexpr int64_t kChunkIn = 512LL << 20, kChunkOut = 1024LL << 20, kChunkNnz = 32LL << 20;
static int64_t ChunkRows(int64_t nrow, int64_t in_row_bytes, int64_t per_row) {      // in_row_bytes 0: nothing staged
  return std::max<int64_t>(1, std::min({nrow, in_row_bytes > 0 ? kChunkIn / in_row_bytes : nrow, kChunkOut / (std::max<int64_t>(per_row, 1) * 8)}));
}
static int Grid(int64_t threads) { return static_cast<int>(std::min<int64_t>((threads + 255) / 256, static_cast<int64_t>(DeviceSMs()) * 16)); }

void Predictor::UploadForest() {
  if (forest_ && forest_->trees == model_.trees.size()) return;
  forest_.reset(new ForestBufs());
  ForestBufs& f = *forest_;
  const size_t T = model_.trees.size();
  std::vector<int> toff(T + 1, 0), loff(T + 1, 0), nl(T), sf, dt, lc, rc, cbeg, clen;
  std::vector<unsigned> cwords;
  std::vector<double> thr, lv, ncnt, lcnt, expv(T, 0.0);
  for (size_t t = 0; t < T; ++t) {
    const HostTree& tr = *model_.trees[t];
    nl[t] = tr.num_leaves;
    expv[t] = tr.ExpectedValue();
    if (tr.num_leaves > 1) f.max_depth = std::max(f.max_depth, tr.MaxDepth());
    toff[t + 1] = toff[t] + std::max(tr.num_leaves - 1, 0);
    loff[t + 1] = loff[t] + tr.num_leaves;
    for (int i = 0; i < tr.num_leaves - 1; ++i) {
      sf.push_back(tr.split_feature[i]); dt.push_back(tr.decision_type[i]); lc.push_back(tr.left_child[i]); rc.push_back(tr.right_child[i]);
      thr.push_back(tr.threshold[i]); ncnt.push_back(tr.internal_count[i]);
      if (tr.decision_type[i] & 1) {
        const int ci = static_cast<int>(tr.threshold[i]);
        cbeg.push_back(static_cast<int>(cwords.size())); clen.push_back(tr.cat_boundaries[ci + 1] - tr.cat_boundaries[ci]);
        for (int w = tr.cat_boundaries[ci]; w < tr.cat_boundaries[ci + 1]; ++w) cwords.push_back(tr.cat_threshold[w]);
      } else { cbeg.push_back(0); clen.push_back(0); }
    }
    for (int i = 0; i < tr.num_leaves; ++i) { lv.push_back(tr.leaf_value[i]); lcnt.push_back(tr.leaf_count[i]); }
  }
  if (!stream_) stream_ = AcquireStream();
  auto up = [&](auto& d, const auto& h) { d.Alloc(std::max<size_t>(h.size(), 1)); if (!h.empty()) d.Upload(h.data(), h.size(), stream_); };
  up(f.tree_offset, toff); up(f.leaf_offset, loff); up(f.num_leaves, nl); up(f.split_feature, sf); up(f.decision_type, dt);
  up(f.left_child, lc); up(f.right_child, rc); up(f.threshold, thr); up(f.leaf_value, lv); up(f.cat_begin, cbeg); up(f.cat_len, clen);
  up(f.node_count, ncnt); up(f.leaf_count, lcnt); up(f.expected, expv); up(f.cat_words, cwords);
  B200_CUDA(cudaStreamSynchronize(stream_));
  f.trees = T;
}

const Predictor::SlotBufs& Predictor::UploadSlots(int t0, int t1) {
  ForestBufs& fb = *forest_;
  if (fb.slots && fb.slots->t0 == t0 && fb.slots->t1 == t1) return *fb.slots;
  std::unique_ptr<SlotBufs> sl(new SlotBufs());
  sl->t0 = t0; sl->t1 = t1;
  const int nfeat = model_.max_feature_idx + 1;
  std::vector<int> slot_of(nfeat, -1), feature_of, split;
  for (int t = t0; t < t1; ++t) {
    const HostTree& tr = *model_.trees[t];
    for (int i = 0; i < tr.num_leaves - 1; ++i) slot_of[tr.split_feature[i]] = 0;
  }
  for (int j = 0; j < nfeat; ++j)
    if (slot_of[j] == 0) { slot_of[j] = static_cast<int>(feature_of.size()); feature_of.push_back(j); }
  for (size_t t = 0; t < model_.trees.size(); ++t) {      // node order of UploadForest; trees outside [t0, t1) are not walked
    const HostTree& tr = *model_.trees[t];
    const bool in = static_cast<int>(t) >= t0 && static_cast<int>(t) < t1;
    for (int i = 0; i < tr.num_leaves - 1; ++i) split.push_back(in ? slot_of[tr.split_feature[i]] : 0);
  }
  sl->U = static_cast<int>(feature_of.size());
  auto up = [&](DevBuf<int>& d, const std::vector<int>& h) { d.Alloc(std::max<size_t>(h.size(), 1)); if (!h.empty()) d.Upload(h.data(), h.size(), stream_); };
  up(sl->slot_of_feature, slot_of); up(sl->feature_of_slot, feature_of); up(sl->split_slot, split);
  B200_CUDA(cudaStreamSynchronize(stream_));
  fb.slots = std::move(sl);
  return *fb.slots;
}

// TreeSHAP scratch of k_predict_contrib: per thread (depth+2)(depth+3)/2 path elements + depth+3 stack frames
struct ShapScratch {
  static constexpr int kThreads = 128;
  int grid = 0, path_stride = 0, frame_stride = 0;
  DevBuf<ShapPathElem> paths;
  DevBuf<ShapFrame> frames;
  ShapScratch(int max_depth, int64_t rows, int sms) {
    const int md = max_depth + 2;
    path_stride = md * (md + 1) / 2 + md;
    frame_stride = md + 2;
    grid = static_cast<int>(std::min<int64_t>((rows + kThreads - 1) / kThreads, static_cast<int64_t>(sms) * 4));
    paths.Alloc(static_cast<size_t>(grid) * kThreads * path_stride);
    frames.Alloc(static_cast<size_t>(grid) * kThreads * frame_stride);
  }
};

// k_predict_raw_es with a group of G lanes per row: one lane for K == 1, the next power of two up to 32 for K <= 32, a warp beyond.
// One group per row of the chunk (no grid-stride reuse): every group of a warp starts at the first iteration and walks the same tree
// index as the others until it stops, so the still-active rows of a warp stay converged.  A group that took a second row after its
// first stopped would walk other trees than its warp neighbours, and the warp would run both walks one after the other.
template <typename T>
void Predictor::LaunchRawEarlyStop(const ForestDev& f, const T* X, int64_t rows, int ncol, int K, int i0, int i1, const EarlyStop& es, double* y) {
  const int G = K == 1 ? 1 : K <= 2 ? 2 : K <= 4 ? 4 : K <= 8 ? 8 : K <= 16 ? 16 : 32;
  const int grid = static_cast<int>((rows * G + 255) / 256);
  switch (G) {
    case 1: k_predict_raw_es<T, 1><<<grid, 256, 0, stream_>>>(f, X, rows, ncol, K, i0, i1, es.freq, es.margin, y); break;
    case 2: k_predict_raw_es<T, 2><<<grid, 256, 0, stream_>>>(f, X, rows, ncol, K, i0, i1, es.freq, es.margin, y); break;
    case 4: k_predict_raw_es<T, 4><<<grid, 256, 0, stream_>>>(f, X, rows, ncol, K, i0, i1, es.freq, es.margin, y); break;
    case 8: k_predict_raw_es<T, 8><<<grid, 256, 0, stream_>>>(f, X, rows, ncol, K, i0, i1, es.freq, es.margin, y); break;
    case 16: k_predict_raw_es<T, 16><<<grid, 256, 0, stream_>>>(f, X, rows, ncol, K, i0, i1, es.freq, es.margin, y); break;
    default: k_predict_raw_es<T, 32><<<grid, 256, 0, stream_>>>(f, X, rows, ncol, K, i0, i1, es.freq, es.margin, y); break;
  }
}

// The chunk loop of dense and CSR input: chunk [r0, end(r0)) has at most `chunk` rows.  stage(r0, rows, launch, dout) puts the chunk's
// rows on the device and calls launch(f, X, data_type, rows, ncol, F1, y), which enqueues the predict kernel of predict_type on X
// [rows][ncol] into y (contributions: [rows][K][F1], zero-filled here).  Each chunk's dout is copied out and waited for.  last_ms spans
// the loop; the rf averaging and the objective transform run on the host after it.
template <typename End, typename Stage>
int64_t Predictor::Run(int64_t nrow, int64_t chunk, int64_t per_row, int predict_type, int t0, int t1, const EarlyStop& es, double* out, End end,
                       Stage stage) {
  const int Kc = model_.num_tree_per_iteration;
  const int64_t rows_max = std::min(chunk, nrow);
  ShapScratch shap(forest_->max_depth, predict_type == 3 ? rows_max : 0, DeviceSMs());
  auto launch = [&](const ForestDev& f, const void* X, int data_type, int64_t rows, int ncol, int F1, double* y) {
    const int64_t width = predict_type == 3 ? static_cast<int64_t>(Kc) * F1 : per_row;
    if (rows * width == 0) return;
    const int grid = Grid(rows * width);
    const float* xf = static_cast<const float*>(X);
    const double* xd = static_cast<const double*>(X);
    if (predict_type == 3) {
      B200_CUDA(cudaMemsetAsync(y, 0, static_cast<size_t>(rows) * width * sizeof(double), stream_));
      if (data_type == 0) k_predict_contrib<float><<<shap.grid, ShapScratch::kThreads, 0, stream_>>>(f, xf, rows, ncol, Kc, t0, t1, F1, shap.paths.p, shap.path_stride, shap.frames.p, shap.frame_stride, y);
      else k_predict_contrib<double><<<shap.grid, ShapScratch::kThreads, 0, stream_>>>(f, xd, rows, ncol, Kc, t0, t1, F1, shap.paths.p, shap.path_stride, shap.frames.p, shap.frame_stride, y);
    } else if (predict_type == 2) {
      if (data_type == 0) k_predict_leaf<float><<<grid, 256, 0, stream_>>>(f, xf, rows, ncol, t0, t1, y);
      else k_predict_leaf<double><<<grid, 256, 0, stream_>>>(f, xd, rows, ncol, t0, t1, y);
    } else if (es.on()) {
      if (data_type == 0) LaunchRawEarlyStop(f, xf, rows, ncol, Kc, t0 / Kc, t1 / Kc, es, y);
      else LaunchRawEarlyStop(f, xd, rows, ncol, Kc, t0 / Kc, t1 / Kc, es, y);
    } else {
      if (data_type == 0) k_predict_raw<float><<<grid, 256, 0, stream_>>>(f, xf, rows, ncol, Kc, t0, t1, y);
      else k_predict_raw<double><<<grid, 256, 0, stream_>>>(f, xd, rows, ncol, Kc, t0, t1, y);
    }
    B200_CUDA(cudaGetLastError());
  };
  DevBuf<double> dout; dout.Alloc(static_cast<size_t>(rows_max) * per_row);
  StreamTimer timer(stream_);
  for (int64_t r0 = 0, r1; r0 < nrow; r0 = r1) {
    r1 = end(r0);
    stage(r0, r1 - r0, launch, dout.p);
    B200_CUDA(cudaMemcpyAsync(out + r0 * per_row, dout.p, static_cast<size_t>(r1 - r0) * per_row * sizeof(double), cudaMemcpyDeviceToHost, stream_));
    B200_CUDA(cudaStreamSynchronize(stream_));
  }
  last_ms = timer.Ms();
  if (predict_type < 2) model_.ConvertScores(out, nrow, Kc, 1, (t1 - t0) / Kc, predict_type == 1);
  return nrow * per_row;
}

int64_t Predictor::PredictMat(const void* data, int data_type, int64_t nrow, int ncol, int predict_type, int start_iteration, int num_iteration,
                              const EarlyStop& es, double* out) {
  EnsureDevice();
  if (data_type != 0 && data_type != 1) Fatal("PredictBatch: unknown data type");
  if (predict_type < 0 || predict_type > 3) Fatal("PredictBatch: unknown predict type");
  if (ncol < model_.max_feature_idx + 1) Fatal("PredictBatch: the matrix has fewer columns than the model has features");
  UploadForest();
  int t0, t1;
  model_.IterRange(start_iteration, num_iteration, &t0, &t1);
  const size_t esz = data_type == 0 ? 4 : 8;
  const bool on_device = IsDevicePointer(data);
  const int64_t per_row = model_.NumPredictPerRow(predict_type, start_iteration, num_iteration);
  const int64_t chunk = ChunkRows(nrow, on_device ? 0 : static_cast<int64_t>(ncol) * esz, per_row);
  DevBuf<unsigned char> xin;
  if (!on_device) xin.Alloc(static_cast<size_t>(chunk) * ncol * esz);
  return Run(nrow, chunk, per_row, predict_type, t0, t1, es, out, [&](int64_t r0) { return std::min(nrow, r0 + chunk); },
             [&](int64_t r0, int64_t rows, auto& launch, double* dout) {
    const void* x = static_cast<const unsigned char*>(data) + static_cast<size_t>(r0) * ncol * esz;
    if (!on_device) { B200_CUDA(cudaMemcpyAsync(xin.p, x, static_cast<size_t>(rows) * ncol * esz, cudaMemcpyHostToDevice, stream_)); x = xin.p; }
    launch(forest_->View(), x, data_type, rows, ncol, model_.max_feature_idx + 2, dout);      // contributions: one per feature + the expected value
  });
}

int64_t Predictor::PredictCSR(const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr,
                              int64_t nelem, int predict_type, int start_iteration, int num_iteration, const EarlyStop& es, double* out) {
  if (indptr_type != 2 && indptr_type != 3) Fatal("PredictBatchCSR: indptr must be INT32 or INT64");
  if (data_type != 1) Fatal("PredictBatchCSR: CSR values must be FLOAT64");
  if (predict_type < 0 || predict_type > 3) Fatal("PredictBatchCSR: unknown predict type");
  if (nindptr < 1) Fatal("PredictBatchCSR: nindptr must be at least 1");
  auto ptr = [&](int64_t i) -> int64_t {
    return indptr_type == 2 ? static_cast<const int32_t*>(indptr)[i] : static_cast<const int64_t*>(indptr)[i];
  };
  if (ptr(0) < 0) Fatal("PredictBatchCSR: indptr[0] is negative");
  for (int64_t i = 1; i < nindptr; ++i)
    if (ptr(i) < ptr(i - 1)) Fatal("PredictBatchCSR: indptr decreases at position " + std::to_string(i));
  if (ptr(nindptr - 1) > nelem) Fatal("PredictBatchCSR: indptr[nindptr-1] is larger than nelem");
  EnsureDevice();
  UploadForest();
  int t0, t1;
  model_.IterRange(start_iteration, num_iteration, &t0, &t1);
  const SlotBufs& sl = UploadSlots(t0, t1);
  ForestDev f = forest_->View();
  f.split_feature = sl.split_slot.p;
  const int U = sl.U;
  const int Kc = model_.num_tree_per_iteration;
  const int F1 = model_.max_feature_idx + 2;
  const int64_t nrow = nindptr - 1;
  // chunks of rows bounded like dense ones (slots as the input matrix, and the output), and by the nonzeros uploaded at once; a row with
  // more nonzeros than that bound is a chunk of its own
  const int64_t per_row = model_.NumPredictPerRow(predict_type, start_iteration, num_iteration);
  const int64_t chunk = ChunkRows(nrow, std::max(U, 1) * 8LL, per_row);
  auto end = [&](int64_t r0) {
    int64_t lo = r0 + 1, hi = std::min(nrow, r0 + chunk);
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) / 2;
      if (ptr(mid) - ptr(r0) <= kChunkNnz) lo = mid; else hi = mid - 1;
    }
    return lo;
  };
  int64_t max_nnz = 0;
  for (int64_t r0 = 0, r1; r0 < nrow; r0 = r1) { r1 = end(r0); max_nnz = std::max(max_nnz, ptr(r1) - ptr(r0)); }
  const int64_t rows_max = std::min(chunk, nrow);
  DevBuf<long long> d_ptr; d_ptr.Alloc(static_cast<size_t>(rows_max) + 1);
  DevBuf<int> d_idx; d_idx.Alloc(static_cast<size_t>(max_nnz));
  DevBuf<double> d_val; d_val.Alloc(static_cast<size_t>(max_nnz));
  DevBuf<double> xs; xs.Alloc(static_cast<size_t>(rows_max) * U);
  DevBuf<double> dslot; dslot.Alloc(predict_type == 3 ? static_cast<size_t>(rows_max) * Kc * (U + 1) : 0);      // contributions per slot
  std::vector<long long> hptr(static_cast<size_t>(rows_max) + 1);
  return Run(nrow, chunk, per_row, predict_type, t0, t1, es, out, end, [&](int64_t r0, int64_t rows, auto& launch, double* dout) {
    const int64_t a = ptr(r0), nnz = ptr(r0 + rows) - a;
    for (int64_t i = 0; i <= rows; ++i) hptr[i] = ptr(r0 + i) - a;
    d_ptr.Upload(hptr.data(), static_cast<size_t>(rows) + 1, stream_);
    if (nnz > 0) {
      d_idx.Upload(indices + a, static_cast<size_t>(nnz), stream_);
      d_val.Upload(static_cast<const double*>(data) + a, static_cast<size_t>(nnz), stream_);
    }
    if (U > 0) {
      k_csr_to_slots<<<Grid(rows * 32), 256, 0, stream_>>>(d_ptr.p, d_idx.p, d_val.p, rows, sl.slot_of_feature.p, F1 - 1, U, xs.p);
      B200_CUDA(cudaGetLastError());
    }
    if (predict_type == 3) {
      launch(f, xs.p, 1, rows, U, U + 1, dslot.p);
      B200_CUDA(cudaMemsetAsync(dout, 0, static_cast<size_t>(rows) * per_row * sizeof(double), stream_));
      k_contrib_slots_to_features<<<Grid(rows * Kc * (U + 1)), 256, 0, stream_>>>(dslot.p, rows * Kc, U, sl.feature_of_slot.p, F1, dout);
      B200_CUDA(cudaGetLastError());
    } else {
      launch(f, xs.p, 1, rows, U, F1, dout);
    }
  });
}

}  // namespace b200gbm
