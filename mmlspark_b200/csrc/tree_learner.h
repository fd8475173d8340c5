// Tree learner of a training Booster: grows one tree on the device from (g, h) and hands it back.  It owns everything a tree is
// built with: the quantised (g,h) words, the histogram slot and pool (K4), the scans (K5), the partition (K7) with its column copy or
// column cache, the controller state, the device tree blob with its pinned host mirror, the ColSampler and the leaf-renewal buffers.
// The Booster keeps the scores, the row sampling and the boosting modes, and applies the grown tree to its scores.
// Part of engine.cu's translation unit (tree_learner.cu is included there).
#pragma once
#include "engine.h"

namespace b200gbm {

class TreeLearner {
 public:
  // cfg is the booster's, read live (ResetConfig refreshes the split parameters copied from it); stream and timing are the booster's
  TreeLearner(const Dataset& train, const Config& cfg, const Objective& obj, bool parallel, bool same_device, int num_sms,
              cudaStream_t stream, Booster::Timing& timing);
  ~TreeLearner();
  void ResetConfig(const Config& cfg);      // the split parameters a ResetParameter may change
  // forced splits: the plan every later tree starts with (forced_splits.h), empty for none; uploaded when it changes
  void SetForcedPlan(const std::vector<ForcedNode>& plan);
  bool HasForcedPlan() const { return !forced_host_.empty(); }

  // the rows a bagged tree is grown on: the in-bag flags and the ascending in-bag row list
  struct Bag { const uint8_t* in_bag; const int* rows; int count; };
  // enqueues the whole leaf-wise growth of one tree on (g, h) without a host sync; bag null: every row.  tree_index (iteration * trees
  // per iteration + class) keys the draws of quantised training's stochastic rounding.
  void Grow(const float* g, const float* h, bool const_hessian, const Bag* bag, int tree_index);
  // quant_train_renew_leaf: the grown tree's leaf values from the leaves' true in-bag sums of the (g, h) it was grown on
  void RenewQuantized(const float* g, const float* h, bool const_hessian);
  // percentile objectives: patch the grown tree's leaf values (score_k null: residuals against rf_pred)
  void Renew(const Objective& obj, const double* score_k, double rf_pred);
  // score_k[row] += shrinkage * leaf value of the row's leaf, walking the leaves' row lists (every row is in a leaf)
  void AddScore(double* score_k, double shrinkage);
  const TreeDev& Tree() const { return tree_dev_; }                 // the grown tree on the device
  const DevBuf<unsigned char>& Blob() const { return tree_blob_; }   // the same tree as one buffer (DART stores copies of it)
  TreeDev TreeAt(unsigned char* blob) const;                          // the fields of such a buffer or copy
  // copies the tree to the host (D2H + sync), converts it, and updates the column cache
  void ReadTree(HostTree* out);

  bool profile_hist = false;                 // time K4 with events on the stream (Timing::hist_ms)
  size_t ColumnCopyBytes() const { return bins_cols_.n; }
  void GetColumnCacheInfo(int64_t* out4) const;
  // {histogram bytes all-reduced, vote record bytes all-gathered (all ranks' records), split rounds enqueued (num_leaves - 1 per tree)}
  void GetCommInfo(int64_t* out3) const { out3[0] = comm_hist_bytes_; out3[1] = comm_rec_bytes_; out3[2] = comm_splits_; }

 private:
  void ResetFeaturesByTree();
  void SeedExtraStreams(const Config& cfg);
  void LaunchPartition(int grid, int last);
  void EnsureColumnCopy();
  void UpdateColumnCache(const HostTree& t);

  const Dataset& train_;
  const Config& cfg_;
  const bool parallel_, same_device_;
  const bool voting_;            // parallel_ and tree_learner=voting: the voting-parallel split chain (kernels.cuh k_scan, k_vote_pack)
  const int num_sms_;
  cudaStream_t stream_;
  Booster::Timing& timing_;
  SplitParams sp_{};
  bool extra_trees_ = false;     // cfg.extra_trees as of the last ResetConfig: launch the scans' extra_trees instantiations
  bool monotone_ = false;        // cfg.monotone_constraints non-empty as of the last ResetConfig: launch the scans' kMono instantiations
  double monotone_penalty_ = 0.0;
  bool smooth_ = false;          // path_smooth > kPathSmoothEps as of the last ResetConfig: launch the kMono instantiations too
  std::vector<signed char> mono_host_;      // [nf_pad] each inner feature's monotone constraint, as uploaded to mono_
  DevBuf<signed char> mono_;
  std::vector<unsigned long long> sets_of_host_;      // [nf_pad] each inner feature's interaction-constraint sets, as uploaded to sets_of_
  DevBuf<unsigned long long> sets_of_;
  bool bynode_ = false;            // feature_fraction_bynode < 1 as of the last ResetConfig: the k_scan grid's sampler column
  int bynode_k_ = 0;               // its sample size K
  DevBuf<uint8_t> node_mask_;      // per-node feature sampling: [2][nf_pad] the round's leaf samples (kernels.cuh d_bynode_sample)
  DevBuf<int> node_work_;          // [2][4][nf_pad] the sampler's scratch
  DevBuf<int> real_order_;         // [nf_pad] Dataset::sample_order: the used features in real-index order
  std::vector<ForcedNode> forced_host_;      // forced splits: the plan as uploaded to forced_, empty for none
  DevBuf<ForcedNode> forced_;
  DevBuf<SplitCand> forced_evals_;           // [plan nodes] each node's evaluation (kernels.cuh d_forced_eval), zeroed before each tree
  int rows_ = 0;                 // rows of the tree being grown (the bag's count when bagged)
  // device state of the tree being grown
  DevBuf<int4> qgh_, qord_;      // per-row fixed-point (g,h) words; the same in leaf order for the leaf being built
  DevBuf<int> idx0_, idx1_;
  DevBuf<long long> quant_sums_;   // quant_train_renew_leaf: [num_leaves][2] the leaves' true sums on K3's fixed-point grid
  DevBuf<long long> H_;          // scratch histogram of the current smaller leaf
  DevBuf<long long> pool_;       // [num_leaves] leaf histograms
  size_t slot_elems_ = 0;
  DevBuf<uint8_t> flags_;        // [num_leaves][nf_pad]
  DevBuf<SplitCand> cands_;      // [2][nf_pad]
  DevBuf<unsigned> xrand_;       // extra_trees: [nf_pad] stream state per feature, then [2][nf_pad] draws of the round (kernels.cuh d_lcg_next)
  DevBuf<int> xrand_pos_;        // [nf_pad] each inner feature's position among the used features in real-index order (its stream's seed offset)
  // voting: top_k clamped to the used features; this rank's [2][top_k] records, every rank's [R][2][top_k], the voted features [2][top_k],
  // and the packed buffer that is all-reduced (kVoteTotals + 2 * top_k storage columns)
  int top_k_ = 0;
  DevBuf<VoteRec> recs_, all_recs_;
  DevBuf<int> voted_;
  DevBuf<long long> packed_;
  long long comm_hist_bytes_ = 0, comm_rec_bytes_ = 0, comm_splits_ = 0;
  DevBuf<LeafState> leaves_;
  DevBuf<TreeCtrl> ctrl_;
  DevBuf<unsigned char> tree_blob_;
  TreeDev tree_dev_{};
  unsigned char* tree_host_ = nullptr;   // pinned mirror of tree_blob_
  TreeCtrl* ctrl_host_ = nullptr;        // pinned
  DevBuf<unsigned> part_bits_;
  DevBuf<int> part_chunks_;
  int part_max_blocks_ = 0;
  // optional [column][row] copies of the uint8 tiles' storage columns for the partition kernel: all of them (full copy), or a pool of
  // slots that UpdateColumnCache fills with the columns the trees split on (column cache)
  DevBuf<uint8_t> bins_cols_;
  size_t cols_stride_ = 0;
  bool cols_tried_ = false;
  DevBuf<int> col_slot_;                   // [num_tiles * 32] slot of each storage column in bins_cols_, -1: not copied
  std::vector<int> col_slot_host_;
  std::vector<int> slot_col_;              // column cache: storage column held by each slot, -1: free (empty for the full copy)
  std::vector<long long> col_splits_;      // column cache: splits on each storage column so far
  long long cache_builds_ = 0, cache_evictions_ = 0;
  LcgRandom col_rand_{2};                  // ColSampler (feature_fraction; the device continues it within a tree for feature_fraction_bynode)
  std::vector<uint8_t> feature_used_host_;
  DevBuf<uint8_t> feature_used_;
  // percentile objectives: sort buffers of the renewal pass (renew_kernel.cuh)
  DevBuf<unsigned long long> rn_keys_a_, rn_keys_b_;
  DevBuf<unsigned> rn_pos_a_, rn_pos_b_, rn_leaf_of_pos_, rn_leaf_a_, rn_leaf_b_;
  DevBuf<double> rn_res_, rn_cdf_, rn_out_;      // rn_out_: [2][num_leaves] outputs, has-rows flags
  DevBuf<int> rn_row_, rn_seg_;
  DevBuf<unsigned char> rn_tmp_;
  size_t rn_tmp_bytes_ = 0;
  // B200GBM_SPLIT_TIMING=1 (debug): events of the tree being grown, per-operation sums reported on stderr at destruction
  std::vector<cudaEvent_t> split_events_, hist_events_;
  std::map<std::string, double> split_op_ms_;
  int split_op_trees_ = 0;
};

}  // namespace b200gbm
