// b200gbm engine: device dataset, data-parallel network state, booster (the GBDT driver; its tree learner is in tree_learner.h).
// Everything below the C ABI (include/b200gbm_c_api.h).  One host thread drives one
// (network, dataset, booster) triple, exactly like one Spark task thread in the reference
// (SURVEY.md fact 8): network / device / last-error state are thread_local.
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>

#include <cstdint>
#include <memory>
#include <stdexcept>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "bin_mapper.h"
#include "bundle.h"
#include "config.h"
#include "kernels.cuh"
#include "model.h"

namespace b200gbm {

#define B200_CUDA(x)                                                                                      \
  do {                                                                                                    \
    cudaError_t e__ = (x);                                                                                \
    if (e__ != cudaSuccess)                                                                               \
      throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(e__) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
  } while (0)
#define B200_NCCL(x)                                                                                      \
  do {                                                                                                    \
    ncclResult_t r__ = (x);                                                                               \
    if (r__ != ncclSuccess)                                                                               \
      throw std::runtime_error(std::string("NCCL error: ") + ncclGetErrorString(r__) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
  } while (0)

[[noreturn]] inline void Fatal(const std::string& m) { throw std::runtime_error(m); }

// ---- per-thread device + network state -------------------------------------------------------
struct SameDeviceComm;          // engine.cu: rank-threads of one process on one device
// The data-parallel communicator of one rank.  NetworkInit picks the backend from the layout it observes: NCCL when every rank has its
// own device, the same-device communicator when every rank is a thread of this process on one device.  Every collective of the engine
// goes through AllReduce / AllGather, which make the same NCCL calls as before on the NCCL backend.
struct Network {
  bool active = false;
  int rank = 0, world = 1;
  ncclComm_t comm = nullptr;
  std::shared_ptr<SameDeviceComm> same_device;
  // in place on `count` elements of buf; (type, op) in (double: sum / max / min), (int64: sum), (uint32: max)
  void AllReduce(void* buf, size_t count, ncclDataType_t type, ncclRedOp_t op, cudaStream_t s) const;
  // recv[r * bytes, (r + 1) * bytes) = rank r's send, on every rank
  void AllGather(const void* send, void* recv, size_t bytes, cudaStream_t s) const;
};
Network& Net();                 // thread-local
int CurrentDevice();            // thread-local CUDA ordinal (selects on first use)
void SetThreadDevice(int ordinal);
void EnsureDevice();            // cudaSetDevice(CurrentDevice()) + fail loudly when no GPU
int DeviceSMs();                // multiprocessor count of CurrentDevice() (grid sizes of the grid-stride kernels)
void NetworkInit(const char* machines, int local_listen_port, int listen_time_out_sec, int num_machines);
void NetworkFree();
void AllReduceHost(double* v, int n, ncclRedOp_t op, cudaStream_t s);      // small host-value collectives, staged through device memory
// The stream of a new dataset or booster on CurrentDevice().  With the same-device communicator it is the one process-wide stream of
// the device, so the ranks' kernels run one after another (k_partition's cooperative grid needs the whole device) and the collectives
// are ordered by the stream alone; that stream lives until the process ends, so objects may outlive LGBM_NetworkFree.
cudaStream_t AcquireStream();
void ReleaseStream(cudaStream_t s);      // destroys a stream of AcquireStream unless it is a shared one

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { Free(); }
  void Alloc(size_t count) {
    Free();
    n = count;
    if (count) B200_CUDA(cudaMalloc(reinterpret_cast<void**>(&p), count * sizeof(T)));
  }
  void Free() { if (p) { cudaFree(p); p = nullptr; } n = 0; }
  void Zero(cudaStream_t s) { if (p) B200_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), s)); }
  void Upload(const T* h, size_t count, cudaStream_t s) { B200_CUDA(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, s)); }
  void Download(T* h, size_t count, cudaStream_t s) const { B200_CUDA(cudaMemcpyAsync(h, p, count * sizeof(T), cudaMemcpyDeviceToHost, s)); }
};

// ---- dataset -----------------------------------------------------------------------------------
class Dataset {
 public:
  ~Dataset();
  // One dataset from nmat row parts that count as one matrix: part 0's rows, then part 1's, ...  Bins, bundles and mappers equal those
  // of one matrix holding the concatenation (a single matrix is nmat = 1), and no host copy of the parts is made.
  // data[i]: host or device pointer (detected per part) of nrow[i] rows; data_type 0=f32 1=f64; reference != null => reuse its bins
  static Dataset* CreateFromMats(int nmat, const void* const* data, int data_type, const int32_t* nrow, int ncol, int is_row_major,
                                 const char* params, const Dataset* reference);
  // the same for nparts host CSR parts; each part has its own indptr, which need not start at 0
  static Dataset* CreateFromCSRs(int nparts, const void* const* indptr, int indptr_type, const int32_t* const* indices, const void* const* data,
                                 int data_type, const int64_t* nindptr, const int64_t* nelem, int64_t num_col, const char* params,
                                 const Dataset* reference);
  // LightGBM streaming ingestion: bins from a column-wise sample, then row blocks pushed in place
  static Dataset* CreateFromSampledColumn(double** sample_data, int** sample_indices, int ncol, const int* num_per_col,
                                          int num_sample_row, int num_total_row, const char* params);
  void PushRows(const void* data, int data_type, int nrow, int ncol, int start_row);
  void GetBinsRowMajor(uint8_t* out) const;                 // fails when a feature has more than 256 bins
  void GetBinsRowMajor16(uint16_t* out) const;
  void GetBinsOfRows(const int32_t* rows, int nrows, uint16_t* out) const;      // [nrows][num_total_features], gathered on the device
  // K4 on this dataset's bins for the given rows (kernel-level parity entry), fp64 [F][256][2] per feature (bundle columns expanded)
  void Histogram(const float* grad, const float* hess, const int32_t* idx, int cnt, double* out) const;
  // quantised training's K3 discretisation (B = bins levels, draws keyed by seed and tree) and packed K4 on the given rows: per row
  // (q_g, q_h) into out_q [num_data][2], the scales (s_g, s_h) into out_scale2, int64 sums of q [F][256][2] per feature into out_hist.
  // hess null: constant hessians (q_h = 1, the count plane).
  struct QuantSpec { int bins = 0; bool stochastic = false; int seed = 0; int tree = 0; };
  void QuantizedHistogram(const float* grad, const float* hess, const int32_t* idx, int cnt, const QuantSpec& quant, int32_t* out_q,
                          double* out_scale2, int64_t* out_hist) const;
  void SetField(const char* name, const void* data, int n, int type);
  void GetField(const char* name, int* out_len, const void** out_ptr, int* out_type) const;
  void SetFeatureNames(const char** names, int n);
  void GetBundles(int* out_num_columns, int* out_column_of) const;      // storage column of every feature (-1: unused)
  // K4's per-block bin-count bound of the uint8 tiles (hist_kernel.cuh): computed from the bins on first use, reused by every
  // booster on this dataset and by Histogram, dropped when rows are binned again.  Safe to call from several host threads.
  RowBlockBound BlockBound() const;
 private:
  std::vector<long long> HistogramInt(const float* grad, const float* hess, const int32_t* idx, int cnt, const QuantSpec& quant,
                                      DevBuf<TreeCtrl>& ctrl, DevBuf<int4>& q) const;
 public:

  int device = 0;
  int num_data = 0, num_total_features = 0;
  Config cfg;
  std::vector<FeatureBins> mappers;          // [num_total_features]
  std::vector<int> used;                     // inner -> real
  std::vector<int> inner_of;                 // real -> inner or -1
  std::vector<FeatMeta> meta_host;
  int nf = 0, nf_pad = 0, num_tiles = 0;
  int nfn = 0, nw = 0;                       // inner features [0, nfn) live in uint8 tiles, [nfn, nf) are wide (> 256 bins, uint16 columns)
  // storage columns of the uint8 tiles: one per plain tile feature and one per feature bundle (bundle.h); without a bundle column = feature
  int num_columns = 0;
  std::vector<std::vector<int>> bundles;     // real indices of the members of each bundle (two or more each)
  std::vector<int> col_feat;                 // [num_tiles * 32] the plain inner feature of a column, -1 for a bundle column or padding
  DevBuf<int> d_col_feat;
  std::vector<int> bundle_base;              // [nf_pad] per inner feature: -1 alone in its column, else its base in a bundle column (d_unbundle)
  DevBuf<int> d_bundle_base;
  DevBuf<BundleMember> d_members;            // members of all bundles, bundle by bundle
  DevBuf<int> d_bundle_start, d_bundle_col;  // [bundles + 1] first member of each bundle, [bundles] its storage column
  size_t hist_pairs = 0;                     // (g,h) pairs of one histogram slot: num_tiles*32*256 for the tiles + the wide features' bins
  std::vector<int> sample_order;             // used features in real-index order -> inner index (ColSampler draws in that order)
  size_t rows_stride = 0;
  DevBuf<uint8_t> bins;                      // [num_tiles][rows_stride][32]
  DevBuf<uint16_t> bins16;                   // [nw][rows_stride]
  const int* BundleBase() const { return bundles.empty() ? nullptr : d_bundle_base.p; }      // null: no feature bundle, no decode
  BinView View() const { return BinView{bins.p, rows_stride, bins16.p, nfn, meta.p, BundleBase()}; }
  DevBuf<FeatMeta> meta;                     // [nf_pad] every inner feature, tile and wide; the wide ones at [nfn, nf)
  // bin tables, one row per feature at its FeatMeta::table_off: [nft][256] for the tile slots, then one row per wide feature
  DevBuf<double> ub;                         // bin upper bounds (categorical: sorted category values)
  DevBuf<uint16_t> catbin;                   // categorical: bin of the i-th sorted category
  bool has_categorical = false;
  std::vector<float> label, weight;
  std::vector<double> init_score;
  std::vector<int32_t> query_boundaries, group_sizes;
  std::vector<int32_t> position;             // display position of each row (any int32 values), empty for none: the ranking objectives' factors
  DevBuf<float> d_label, d_weight;
  DevBuf<int> d_qb, d_position;
  std::vector<std::string> feature_names;
  cudaStream_t stream = nullptr;
  double ingest_ms = 0.0;                    // H2D + binning time of a matrix / CSR create, or the sum over PushRows calls (CUDA events)

 private:
  // every create runs NewShell, SetMappers and AllocBins, in that order
  static std::unique_ptr<Dataset> NewShell(int nrow, int ncol, const char* params);
  // may_bundle: the create path can check every row before binning (matrix and CSR input)
  template <typename Sample> void SetMappers(const Dataset* reference, bool may_bundle, Sample sample);
  // drops every bundle with a row in which two members are away from their most frequent bin; count(conflicts) runs the row check
  template <typename Count> void DissolveConflictingBundles(Count count);
  void UploadBundleMembers();
  std::vector<int> SampleRows() const;
  void AllocBins();
  template <typename T> void UnpackTiles(T* out) const;
  struct MatPart { const void* data; long long nrow; bool on_device; };      // rows of a matrix, one after another
  void BinBlock(const std::vector<MatPart>& parts, int data_type, int is_row_major, long long start_row);
  // fn(device rows, rows, leading dimension, first row counted over all parts) for each block of rows of the parts, in order; host
  // parts are staged through device memory
  template <typename Fn> void ForEachDeviceBlock(const std::vector<MatPart>& parts, int data_type, int is_row_major, Fn fn);
  // persistent H2D staging of the host ingestion path (two device chunks, a copy stream, events); released once every row is in
  DevBuf<unsigned char> ingest_buf_[2];
  cudaStream_t ingest_copy_stream_ = nullptr;
  cudaEvent_t ingest_copied_[2] = {nullptr, nullptr}, ingest_binned_[2] = {nullptr, nullptr};
  long long ingest_rows_done_ = 0;
  void ReleaseIngestStaging();
  void UploadMeta();
  mutable DevBuf<int> block_bound_;          // [num_tiles][bound_blocks(num_data) + 1], empty until BlockBound()
  mutable std::mutex block_bound_mu_;        // boosters on other host threads may ask for the bound at the same time
};

// ---- booster -----------------------------------------------------------------------------------
struct ValidSet {
  const Dataset* ds = nullptr;
  DevBuf<double> score;   // [K][n]
};
class Objective;          // objective.h
class TreeLearner;        // tree_learner.h
class Metrics;            // metrics.h
class Predictor;          // predictor.h

class Booster {
 public:
  Booster(const Dataset* train, const char* params);      // training booster
  explicit Booster(const std::string& model_text);        // prediction-only booster
  ~Booster();

  bool UpdateOneIter();                                   // returns is_finished
  bool UpdateOneIterCustom(const float* grad, const float* hess);
  void ResetParameter(const char* params);
  void AddValidData(const Dataset* valid);
  void MergeFrom(const Booster* other);
  std::vector<std::string> EvalNames() const;
  std::vector<double> GetEval(int data_idx);
  void GetPredict(int data_idx, int64_t* out_len, double* out);
  int64_t NumPredict(int data_idx) const;
  void GetRawScores(int data_idx, double* out);
  // the objective's gradients at the current training scores, class-major [K][n], computed into scratch buffers: the training state
  // (grad_ / hess_, which rf keeps from construction and GOSS rescales in place) is not touched
  void GetGradients(float* grad, float* hess);
  // the ranking objectives' position factors: the distinct position values of the training data (over every rank, sorted) and the
  // factor of each; empty without a position field, for other objectives and for a prediction-only booster
  void GetPositionBias(std::vector<int32_t>* values, std::vector<double>* factors) const;
  // LGBM_BoosterRefit (refit.cu): leaf_preds [nrow][ncol] row-major host memory, the leaf of training row i in model j.  Every check
  // (and with data-parallel ranks every rank's outcome) comes before anything changes, so a failed refit leaves the model as it was.
  void Refit(const int32_t* leaf_preds, int nrow, int ncol);
  struct RefitTiming { double stage_ms = 0, tree_ms = 0; int batches = 0, blocks = 0; };
  RefitTiming refit_timing;      // of the last refit: host time of the staging and of the per-tree work, batches of models, row blocks
  void GetInfo(int* out4) const { out4[0] = parallel_ ? Net().world : 1; out4[1] = parallel_ ? Net().rank : 0; out4[2] = same_device_ ? 3 : 0; out4[3] = const_hessian_ ? 1 : 0; }
  std::string SaveModelToString(int start_iteration, int num_iteration, int importance_type) const;
  std::string DumpModelJson(int start_iteration, int num_iteration) const;

  // instrumentation for bench.py / parity tests (B200GBM_* extensions of the C ABI)
  struct Timing { double hist_ms = 0, total_ms = 0; long long hist_rows = 0; long long hist_launches = 0, launches = 0; };
  Timing timing;
  void SetProfile(bool profile_hist);                     // time K4 with events on the engine stream
  void GetMemoryInfo(int64_t* out2);
  void GetColumnCacheInfo(int64_t* out4) const;
  void GetCommInfo(int64_t* out3) const;

  Config cfg;
  HostModel model;
  const Dataset* train = nullptr;
  std::unique_ptr<Predictor> predictor;      // batched prediction on the device; reads model and stream_, which it acquires when null
  int K = 1;
  int iter = 0;
  int num_init_iteration = 0;

 private:
  void InitTraining();
  bool TrainTrees(const float* custom_g, const float* custom_h);
  void TrainOneTree(int class_id, HostTree* out);
  double BoostFromAverage(int class_id);

  std::unique_ptr<Objective> obj_;      // training boosters only
  std::unique_ptr<TreeLearner> learner_;      // training boosters only; uses stream_, so it is freed before the stream
  std::unique_ptr<Metrics> metrics_;          // training boosters only
  int device_ = 0;
  cudaStream_t stream_ = nullptr;
  bool parallel_ = false;
  bool voting_ = false;                 // parallel_ and tree_learner=voting at create: the learner's split chain, which ResetParameter keeps
  bool same_device_ = false;            // parallel_ over the same-device communicator: all ranks are threads of this process on this device
  bool const_hessian_ = false;
  bool has_init_score_ = false;
  bool custom_grad_ = false;            // trained on custom gradients at least once: refit has no objective to take gradients from
  double shrinkage_ = 0.1;
  // row subsampling: bagging / GOSS / random forest (SURVEY §8f-3)
  bool is_rf_ = false, is_goss_ = false, bagging_ = false, balanced_bagging_ = false, use_bag_ = false, need_re_bagging_ = false;
  int bag_count_ = 0, bag_blocks_ = 0;
  DevBuf<unsigned> bag_lcg_;            // one LCG state per 1024-row block
  DevBuf<LcgJump> bag_jump_;
  DevBuf<uint8_t> in_bag_;
  DevBuf<int> bag_block_cnt_, bag_idx_, bag_total_;
  std::vector<double> rf_init_scores_;
  void Bagging(int it);
  void ComputeGradientsAt(const double* score);
  // DART (SURVEY §8f-3): every trained tree keeps its device blob so dropped trees can be re-applied to the binned data
  bool is_dart_ = false, dart_dropped_this_iter_ = false;
  LcgRandom drop_rand_{4};
  std::vector<int> drop_index_;
  std::vector<double> tree_weight_;
  double sum_weight_ = 0.0;
  std::vector<std::unique_ptr<DevBuf<unsigned char>>> tree_store_;     // [iteration * K + class]
  void DroppingTrees();
  void DartNormalize();
  void AddStoredTree(int iter_index, int class_id, bool to_train, bool to_valid);
  // device state
  DevBuf<double> score_;        // [K][n]
  DevBuf<float> grad_, hess_;   // [K][n]
  std::vector<ValidSet*> valids_;
  // data_idx 0: the training data and its scores, i > 0: validation set i - 1; fails for any other data_idx
  std::pair<const Dataset*, const DevBuf<double>*> ScoredData(int data_idx) const;
  int num_sms_ = 0;
  cudaEvent_t ev_a_ = nullptr, ev_b_ = nullptr;
};

}  // namespace b200gbm
