// TreeLearner (tree_learner.h).  Included by engine.cu: one translation unit with the kernels it launches.
#include "tree_learner.h"

namespace b200gbm {

static size_t Align16(size_t x) { return (x + 15) & ~static_cast<size_t>(15); }
constexpr int kScanSmem = (768 + 64) * 8;         // k_scan: scratch of the categorical split search (one warp per block runs it)
constexpr int kPartTickets = 8;                   // k_partition: chunks a block takes per ticket (0: one chunk per ticket)

// ColSampler's GetCnt: the size of a feature sample ([UPSTREAM] ColSampler::GetCnt)
static int SampleCount(int total, double fraction) { return std::max(static_cast<int>(total * fraction + 0.5), std::min(2, total)); }

// The split scans of one (extra_trees, output-based gains) pair, indexed [extra_trees][monotone constraints or path smoothing].  Each pair
// has its own instantiations, so that the default one compiles to what it was without either.
struct ScanKernels {
  decltype(&k_scan<kScanPlain>) scan;
  decltype(&k_scan_wide<false, false>) scan_wide;
};
static const ScanKernels kScanKernels[2][2] = {
    {{k_scan<kScanPlain, false, false>, k_scan_wide<false, false>}, {k_scan<kScanPlain, false, true>, k_scan_wide<false, true>}},
    {{k_scan<kScanPlain, true, false>, k_scan_wide<true, false>}, {k_scan<kScanPlain, true, true>, k_scan_wide<true, true>}}};

// The device tree blob: the TreeDev fields one after another in this order, each 16-byte aligned, with its element count for L
// leaves.  The allocation, a stored copy (DART) and the pinned host mirror all take their field pointers from this one list.
template <typename Fn>
static void ForEachTreeField(TreeDev& t, int L, Fn fn) {
  const size_t nodes = L - 1, leaves = L;
  fn(t.left_child, nodes); fn(t.right_child, nodes); fn(t.split_feature_inner, nodes); fn(t.threshold_bin, nodes);
  fn(t.decision_type, nodes); fn(t.split_gain, nodes); fn(t.leaf_value, leaves); fn(t.leaf_weight, leaves); fn(t.leaf_count, leaves);
  fn(t.internal_value, nodes); fn(t.internal_weight, nodes); fn(t.internal_count, nodes); fn(t.leaf_parent, leaves);
  fn(t.leaf_depth, leaves); fn(t.num_leaves, 1); fn(t.cat_bits, 8 * nodes); fn(t.cat_list, kCatListMax * nodes); fn(t.cat_list_len, nodes);
}
static size_t TreeBlobBytes(int L) {
  TreeDev t{};
  size_t bytes = 0;
  ForEachTreeField(t, L, [&](auto*& p, size_t count) { bytes += Align16(count * sizeof(*p)); });
  return bytes;
}
static TreeDev TreeBlobAt(unsigned char* base, int L) {
  TreeDev t{};
  size_t off = 0;
  ForEachTreeField(t, L, [&](auto*& p, size_t count) {
    p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + off);
    off += Align16(count * sizeof(*p));
  });
  return t;
}

TreeLearner::TreeLearner(const Dataset& train, const Config& cfg, const Objective& obj, bool parallel, bool same_device, int num_sms,
                         cudaStream_t stream, Booster::Timing& timing)
    : train_(train), cfg_(cfg), parallel_(parallel), same_device_(same_device), voting_(parallel && cfg.tree_learner == "voting"), num_sms_(num_sms),
      stream_(stream), timing_(timing) {
  const int n = train.num_data;
  const int L = cfg.num_leaves;
  // leaf passes gather single 32-byte sectors: ask L2 not to fetch the neighbouring sector from DRAM on a miss (default 64 B).
  // A hint for the sparse leaf passes; streamed passes read whole sectors anyway.
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  cudaGetLastError();
  B200_CUDA(set_k4_smem_limit());
  for (const auto& by_mono : kScanKernels)
    for (const ScanKernels& k : by_mono) {
      B200_CUDA(cudaFuncSetAttribute(k.scan, cudaFuncAttributeMaxDynamicSharedMemorySize, kScanSmem));
      if (train.nw > 0) B200_CUDA(cudaFuncSetAttribute(k.scan_wide, cudaFuncAttributeMaxDynamicSharedMemorySize, kWideMaxBins * 8));
    }
  mono_.Alloc(train.nf_pad);      // allocated whatever monotone_constraints says: a ResetParameter may set them
  sets_of_.Alloc(train.nf_pad);   // and whatever interaction_constraints says
  // and whatever feature_fraction_bynode says: the node masks, the sampler's scratch and the used features in real-index order
  node_mask_.Alloc(2 * static_cast<size_t>(train.nf_pad)); node_work_.Alloc(8 * static_cast<size_t>(train.nf_pad));
  real_order_.Alloc(train.nf_pad); real_order_.Upload(train.sample_order.data(), train.nf, stream_);

  ResetConfig(cfg);
  sp_.num_leaves = L; sp_.parallel = parallel_ ? 1 : 0;
  sp_.nf = train.nf; sp_.nf_pad = train.nf_pad; sp_.num_tiles = train.num_tiles; sp_.nfn = train.nfn;
  {   // categorical split search parameters (Config keeps the native defaults unless given, SURVEY.md B.2)
    sp_.cat_l2 = cfg.cat_l2; sp_.cat_smooth = cfg.cat_smooth;
    sp_.max_cat_threshold = cfg.max_cat_threshold; sp_.max_cat_to_onehot = cfg.max_cat_to_onehot;
    sp_.min_data_per_group = cfg.min_data_per_group;
    if (train.nw > 0) {
      if (sp_.max_cat_threshold > kCatListMax) Fatal("max_cat_threshold > " + std::to_string(kCatListMax) + " is not supported together with categorical features of more than 256 bins");
      if (sp_.max_cat_to_onehot > 256) Fatal("max_cat_to_onehot > 256 is not supported together with categorical features of more than 256 bins");
      B200_CUDA(cudaFuncSetAttribute(k4_hist_wide<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * kWideHistSeg * 4));
      B200_CUDA(cudaFuncSetAttribute(k4_hist_wide<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * kWideHistSeg * 4));
    }
  }

  qgh_.Alloc(n); qord_.Alloc(n); idx0_.Alloc(n); idx1_.Alloc(n);
  quant_sums_.Alloc(2 * static_cast<size_t>(L));      // whatever quant_train_renew_leaf says: a ResetParameter may set it
  slot_elems_ = train.hist_pairs * 2;
  H_.Alloc(slot_elems_); H_.Zero(stream_); pool_.Alloc(slot_elems_ * L);
  {
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_partition, 256, 0));
    int coop = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, CurrentDevice());
    if (!coop || per_sm < 1) Fatal("this device cannot launch the cooperative partition kernel");
    part_max_blocks_ = per_sm * num_sms_;
  }
  flags_.Alloc(static_cast<size_t>(L) * train.nf_pad);
  cands_.Alloc(2 * static_cast<size_t>(train.nf_pad));
  {   // extra_trees streams, allocated whatever extra_trees says: a ResetParameter may turn it on.  The engine's inner order puts the wide
      // features last, so feature sample_order[i] is used feature i in real-index order.
    std::vector<int> pos(train.nf_pad, 0);
    for (int i = 0; i < train.nf; ++i) pos[train.sample_order[i]] = i;
    xrand_pos_.Alloc(train.nf_pad); xrand_pos_.Upload(pos.data(), pos.size(), stream_);
    xrand_.Alloc(3 * static_cast<size_t>(train.nf_pad));
    SeedExtraStreams(cfg);
  }
  if (voting_) {      // Booster checked top_k > 0, no feature of more than 256 bins and R * top_k <= kVoteMaxRecords
    B200_CUDA(cudaFuncSetAttribute(k_scan<kScanLocal>, cudaFuncAttributeMaxDynamicSharedMemorySize, kScanSmem));
    B200_CUDA(cudaFuncSetAttribute(k_scan<kScanGlobal>, cudaFuncAttributeMaxDynamicSharedMemorySize, kScanSmem));
    top_k_ = std::max(1, std::min(cfg.top_k, train.nf));
    recs_.Alloc(2 * static_cast<size_t>(top_k_)); all_recs_.Alloc(2 * static_cast<size_t>(top_k_) * Net().world);
    voted_.Alloc(2 * static_cast<size_t>(top_k_));
    packed_.Alloc(kVoteTotals + 2 * static_cast<size_t>(top_k_) * kVoteColumn); packed_.Zero(stream_);
  }
  leaves_.Alloc(L); ctrl_.Alloc(1); ctrl_.Zero(stream_);
  const int chunks = n / kPartChunk + 2;
  part_bits_.Alloc(static_cast<size_t>(chunks) * (kPartChunk / 32)); part_chunks_.Alloc(static_cast<size_t>(chunks) + chunks / kPartLocalScan + 8); part_chunks_.Zero(stream_);      // + the super-chunk totals of the two-level scan
  const size_t blob_bytes = TreeBlobBytes(L);
  tree_blob_.Alloc(blob_bytes);
  tree_dev_ = TreeAt(tree_blob_.p);
  B200_CUDA(cudaMemsetAsync(tree_blob_.p, 0, blob_bytes, stream_));
  B200_CUDA(cudaMallocHost(reinterpret_cast<void**>(&tree_host_), blob_bytes));
  B200_CUDA(cudaMallocHost(reinterpret_cast<void**>(&ctrl_host_), sizeof(TreeCtrl)));
  if (obj.RenewsLeaves()) {      // sort buffers of the renewal pass (renew_kernel.cuh)
    rn_keys_a_.Alloc(n); rn_keys_b_.Alloc(n); rn_pos_a_.Alloc(n); rn_pos_b_.Alloc(n); rn_leaf_of_pos_.Alloc(n); rn_leaf_a_.Alloc(n); rn_leaf_b_.Alloc(n);
    rn_res_.Alloc(n); rn_row_.Alloc(n); rn_seg_.Alloc(L + 1); rn_out_.Alloc(2 * static_cast<size_t>(L));
    if (obj.RenewWeights()) rn_cdf_.Alloc(n);
    size_t t1 = 0, t2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t1, rn_keys_a_.p, rn_keys_b_.p, rn_pos_a_.p, rn_pos_b_.p, n, 0, 64, stream_);
    cub::DeviceRadixSort::SortPairs(nullptr, t2, rn_leaf_a_.p, rn_leaf_b_.p, rn_pos_b_.p, rn_pos_a_.p, n, 0, 32, stream_);
    rn_tmp_bytes_ = std::max(t1, t2);
    rn_tmp_.Alloc(rn_tmp_bytes_ + 16);
  }
  // ColSampler: one draw at init, then one per tree ([UPSTREAM] ColSampler::SetTrainingData / ResetByTree)
  col_rand_ = LcgRandom(cfg.feature_fraction_seed);
  feature_used_host_.assign(train.nf_pad, 0);
  for (int u = 0; u < train.nf; ++u) feature_used_host_[u] = 1;
  feature_used_.Alloc(train.nf_pad);
  feature_used_.Upload(feature_used_host_.data(), train.nf_pad, stream_);
  ResetFeaturesByTree();
}

TreeLearner::~TreeLearner() {
  if (split_op_trees_ > 0) {
    double tot = 0; for (auto& kv : split_op_ms_) tot += kv.second;
    fprintf(stderr, "[b200gbm split timing] %d trees, %.3f ms per tree in split operations:", split_op_trees_, tot / split_op_trees_);
    for (auto& kv : split_op_ms_) fprintf(stderr, " %s=%.1fus", kv.first.c_str(), 1000.0 * kv.second / split_op_trees_ / std::max(cfg_.num_leaves - 1, 1));
    fprintf(stderr, " (per split)\n");
  }
  if (tree_host_) cudaFreeHost(tree_host_);
  if (ctrl_host_) cudaFreeHost(ctrl_host_);
}

void TreeLearner::ResetConfig(const Config& cfg) {
  sp_.l1 = cfg.lambda_l1; sp_.l2 = cfg.lambda_l2; sp_.max_delta_step = cfg.max_delta_step; sp_.min_gain_to_split = cfg.min_gain_to_split;
  sp_.min_sum_hessian = cfg.min_sum_hessian_in_leaf; sp_.min_data_in_leaf = cfg.min_data_in_leaf; sp_.max_depth = cfg.max_depth;
  extra_trees_ = cfg.extra_trees;
  SeedExtraStreams(cfg);      // [UPSTREAM] HistogramPool::ResetConfig re-runs SetFeatureInfo, which re-seeds every feature's Random
  // monotone constraints: a non-empty list runs the constrained scans for every feature, even when every entry is 0 ([UPSTREAM] USE_MC).
  // The list is indexed by real feature (Booster checked its length and entries); the device copy by inner feature.  Uploaded here when
  // it changes, ordered after the trees already enqueued (a learning-rate delegate resets every iteration and uploads nothing).
  monotone_ = !cfg.monotone_constraints.empty();
  monotone_penalty_ = cfg.monotone_penalty;
  std::vector<signed char> types(train_.nf_pad, 0);
  if (monotone_)
    for (int u = 0; u < train_.nf; ++u) types[u] = static_cast<signed char>(cfg.monotone_constraints[train_.used[u]]);
  // path smoothing runs the same output-based scans, with all-zero types when there is no list.  Never on for the voting learner
  // (Booster rejects path_smooth for it).
  sp_.path_smooth = cfg.path_smooth;
  smooth_ = !voting_ && cfg.path_smooth > kPathSmoothEps;
  if (types != mono_host_) {
    mono_host_ = std::move(types);
    mono_.Upload(mono_host_.data(), mono_host_.size(), stream_);
  }
  // interaction constraints: sets_of[u] has bit s set when set s holds inner feature u's real index (Booster checked the indices and
  // that there are at most 64 sets).  Uploaded when it changes, as the monotone types are.
  // never on for the voting learner, whose scans do not apply the masks (Booster rejects a list for it)
  sp_.interaction = (voting_ || cfg.interaction_constraints.empty()) ? 0 : 1;
  std::vector<unsigned long long> by_real(train_.num_total_features, 0ull), sets(train_.nf_pad, 0ull);
  for (size_t s = 0; s < cfg.interaction_constraints.size(); ++s)
    for (int f : cfg.interaction_constraints[s]) by_real[f] |= 1ull << s;
  for (int u = 0; u < train_.nf; ++u) sets[u] = by_real[train_.used[u]];
  if (sets != sets_of_host_) {
    sets_of_host_ = std::move(sets);
    sets_of_.Upload(sets_of_host_.data(), sets_of_host_.size(), stream_);
  }
  // per-node feature sampling: K from the size of the tree's sample, which is fixed by feature_fraction.  Never on for the voting
  // learner (Booster rejects feature_fraction_bynode < 1 for it).
  bynode_ = !voting_ && cfg.feature_fraction_bynode < 1.0;
  const int pool = cfg.feature_fraction < 1.0 ? SampleCount(train_.nf, cfg.feature_fraction) : train_.nf;
  bynode_k_ = bynode_ ? SampleCount(pool, cfg.feature_fraction_bynode) : 0;
}

void TreeLearner::SetForcedPlan(const std::vector<ForcedNode>& plan) {
  const bool same = plan.size() == forced_host_.size() &&
                    (plan.empty() || std::memcmp(plan.data(), forced_host_.data(), plan.size() * sizeof(ForcedNode)) == 0);
  if (same) return;
  forced_host_ = plan;
  forced_.Alloc(plan.size()); forced_evals_.Alloc(plan.size());      // frees the old buffers: cudaFree waits for the trees enqueued
  if (!plan.empty()) forced_.Upload(forced_host_.data(), plan.size(), stream_);
}

// extra_trees streams (kernels.cuh d_lcg_next): used feature i in real-index order starts at extra_seed + i.  One small kernel on the
// stream, ordered after the trees already enqueued; nothing is copied from the host.  With extra_trees off the states are never read.
void TreeLearner::SeedExtraStreams(const Config& cfg) {
  if (!xrand_.p || !cfg.extra_trees) return;      // the constructor's first ResetConfig runs before the buffers exist; it seeds after them
  k_extra_seed<<<1, 256, 0, stream_>>>(xrand_.p, xrand_pos_.p, train_.nf, cfg.extra_seed);
  B200_CUDA(cudaGetLastError());
}

TreeDev TreeLearner::TreeAt(unsigned char* blob) const { return TreeBlobAt(blob, sp_.num_leaves); }

void TreeLearner::ResetFeaturesByTree() {
  if (cfg_.feature_fraction >= 1.0) return;
  const int total = train_.nf;
  const int cnt = SampleCount(total, cfg_.feature_fraction);
  std::fill(feature_used_host_.begin(), feature_used_host_.end(), 0);
  for (int i : col_rand_.Sample(total, cnt)) feature_used_host_[train_.sample_order[i]] = 1;      // the draw indexes the used features in real-index order
  // no host sync: the copy is ordered after the previous tree's kernels on the same stream, and a copy from pageable memory is staged
  // by the driver before the call returns, so the host vector may be rewritten for the next tree
  feature_used_.Upload(feature_used_host_.data(), train_.nf_pad, stream_);
}

// [LightGBM SerialTreeLearner::RenewTreeOutput] device pass described in renew_kernel.cuh; patches tree_dev_.leaf_value in place
void TreeLearner::Renew(const Objective& obj, const double* score_k, double rf_pred) {
  const int total = rows_;
  const int L = cfg_.num_leaves;
  cudaStream_t s = stream_;
  TreeCtrl* ctrl = ctrl_.p;
  const int egrid = num_sms_ * 8;
  const float* wptr = obj.RenewWeights();      // null: unweighted
  k_renew_gather<<<egrid, 256, 0, s>>>(ctrl, leaves_.p, idx0_.p, idx1_.p, train_.d_label.p, score_k, rf_pred,
                                       rn_keys_a_.p, rn_pos_a_.p, rn_res_.p, rn_leaf_of_pos_.p, rn_row_.p);
  size_t tb = rn_tmp_bytes_;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(rn_tmp_.p, tb, rn_keys_a_.p, rn_keys_b_.p, rn_pos_a_.p, rn_pos_b_.p, total, 0, 64, s));
  k_renew_leaf_keys<<<egrid, 256, 0, s>>>(rn_pos_b_.p, rn_leaf_of_pos_.p, total, rn_leaf_a_.p);
  int leaf_bits = 1;
  while ((1 << leaf_bits) < L) ++leaf_bits;
  tb = rn_tmp_bytes_;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(rn_tmp_.p, tb, rn_leaf_a_.p, rn_leaf_b_.p, rn_pos_b_.p, rn_pos_a_.p, total, 0, leaf_bits, s));
  k_renew_offsets<<<1, 32, 0, s>>>(ctrl, leaves_.p, rn_seg_.p);
  double* out = rn_out_.p;
  double* has = rn_out_.p + L;
  const int lgrid = (L + 127) / 128;
  if (!wptr) {
    k_renew_unweighted<<<lgrid, 128, 0, s>>>(ctrl, rn_seg_.p, rn_pos_a_.p, rn_res_.p, obj.RenewAlpha(), out, has);
  } else {
    k_renew_cdf<<<L, 1024, 0, s>>>(ctrl, rn_seg_.p, rn_pos_a_.p, rn_row_.p, wptr, rn_cdf_.p);
    k_renew_weighted<<<lgrid, 128, 0, s>>>(ctrl, rn_seg_.p, rn_pos_a_.p, rn_res_.p, rn_cdf_.p, obj.RenewAlpha(), out, has);
  }
  if (parallel_) Net().AllReduce(out, 2 * static_cast<size_t>(L), ncclDouble, ncclSum, s);
  k_renew_apply<<<lgrid, 128, 0, s>>>(ctrl, tree_dev_, out, has, parallel_ ? 1 : 0);
  B200_CUDA(cudaGetLastError());
  timing_.launches += wptr ? 7 : 6;
}

// quant_train_renew_leaf: the leaves' row lists are this rank's in-bag rows, so the sums are all-reduced as the histograms are
void TreeLearner::RenewQuantized(const float* g, const float* h, bool const_hessian) {
  const int L = cfg_.num_leaves;
  cudaStream_t s = stream_;
  B200_CUDA(cudaMemsetAsync(quant_sums_.p, 0, quant_sums_.n * sizeof(long long), s));
  // about 8 blocks per SM in all, at least one per leaf; the grid's x dimension takes any num_leaves
  const int per_leaf = std::max(1, num_sms_ * 8 / L);
  k_quant_leaf_sums<<<static_cast<unsigned>(static_cast<long long>(per_leaf) * L), 256, 0, s>>>(ctrl_.p, leaves_.p, idx0_.p, idx1_.p, g, h,
                                                                                                const_hessian ? 1 : 0, per_leaf, quant_sums_.p);
  if (parallel_) Net().AllReduce(quant_sums_.p, quant_sums_.n, ncclInt64, ncclSum, s);
  k_quant_renew_apply<<<(L + 127) / 128, 128, 0, s>>>(ctrl_.p, tree_dev_, quant_sums_.p, const_hessian ? 1 : 0, sp_);
  B200_CUDA(cudaGetLastError());
  timing_.launches += 2;
}

// k_partition is launched cooperatively: its software grid barriers need every block resident
// Column-major copies of the training tiles for k_partition, so that its phase 1 reads one byte per row instead of a 32-byte sector —
// same results either way.  Set up once, before the first tree, after every other buffer of the booster exists, and only within a
// reserve of device memory (validation scores, metric and prediction scratch come later); B200GBM_COLUMN_COPY=0 disables it.
//   full copy     every storage column (kernels.cuh: k_tiles_to_columns), if it fits
//   column cache  otherwise a pool of as many column slots as fit, filled between trees with the columns the trees split on
//                 (UpdateColumnCache); B200GBM_COLUMN_CACHE_COLUMNS=k forces this mode with at most k slots
// With R ranks on one device (same-device network) all of them reach this point at their first tree, when every rank's training buffers
// exist: they measure the free memory before any of them allocates a copy, and each takes at most 1/R of what lies above the reserve.
void TreeLearner::EnsureColumnCopy() {
  if (cols_tried_) return;
  cols_tried_ = true;
  const Dataset& d = train_;
  const char* env = std::getenv("B200GBM_COLUMN_COPY");
  if ((env && std::atoi(env) == 0) || d.nfn == 0) return;      // the same on every rank: the ranks share the bin layout and the process
  size_t free_b = 0, total_b = 0;
  const bool mem_ok = cudaMemGetInfo(&free_b, &total_b) == cudaSuccess;
  if (!mem_ok) cudaGetLastError();
  size_t share = 1;
  if (same_device_) {
    double arrived = 0.0;
    AllReduceHost(&arrived, 1, ncclSum, stream_);      // every rank built its buffers
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); free_b = 0; }
    double f = mem_ok ? static_cast<double>(free_b) : 0.0;
    AllReduceHost(&f, 1, ncclMin, stream_);            // every rank measured before any allocates
    free_b = static_cast<size_t>(f);
    share = static_cast<size_t>(Net().world);
  }
  if (!mem_ok || d.num_data == 0) return;
  const char* force = std::getenv("B200GBM_COLUMN_CACHE_COLUMNS");
  const size_t stride = (static_cast<size_t>(d.num_data) + 255) & ~static_cast<size_t>(255);
  const int ncols = d.num_tiles * 32;
  const size_t need = static_cast<size_t>(ncols) * stride;
  const size_t reserve = std::max<size_t>(static_cast<size_t>(8) << 30, total_b / 10);
  const size_t spare = free_b > reserve ? (free_b - reserve) / share : 0;
  const bool full = !force && spare >= need;
  int slots = ncols;
  if (!full) {
    slots = static_cast<int>(std::min<size_t>(d.num_columns, spare / stride));
    if (force) slots = std::min(slots, std::max(0, std::atoi(force)));
    if (slots == 0) return;
  }
  const size_t bytes = static_cast<size_t>(slots) * stride;
  uint8_t* p = nullptr;
  if (cudaMalloc(reinterpret_cast<void**>(&p), bytes) != cudaSuccess) { cudaGetLastError(); return; }
  bins_cols_.p = p; bins_cols_.n = bytes;
  cols_stride_ = stride;
  col_slot_host_.assign(ncols, -1);
  if (full) {
    for (int c = 0; c < ncols; ++c) col_slot_host_[c] = c;
    const long long work = ((static_cast<long long>(d.num_data) + 255) / 256) * d.num_tiles;
    k_tiles_to_columns<<<static_cast<unsigned>(std::min<long long>(work, static_cast<long long>(num_sms_) * 16)), 256, 0, stream_>>>(
        d.bins.p, d.rows_stride, d.num_tiles, d.num_data, bins_cols_.p, stride);
    B200_CUDA(cudaGetLastError());
  } else {
    slot_col_.assign(slots, -1);
    col_splits_.assign(ncols, 0);
  }
  col_slot_.Alloc(ncols);
  col_slot_.Upload(col_slot_host_.data(), ncols, stream_);
}

// Column cache, after each tree (its host copy is read back, the stream is idle): count the tree's splits per storage column (wide
// features have their own uint16 columns and are not counted), then copy the most split-on columns that are not cached into free slots.
// When the pool is full, a candidate replaces the least split-on cached column only if that one has fewer splits, so columns that are
// split on often stay.  At most kColumnBuildsMax columns (N x 32 bytes read each) are built per tree, in one launch on the stream;
// the next tree's partitions see the new slot table in stream order, with no host sync inside the tree.
void TreeLearner::UpdateColumnCache(const HostTree& t) {
  if (slot_col_.empty()) return;
  const Dataset& d = train_;
  for (int i = 0; i + 1 < t.num_leaves; ++i) {
    const int f = t.split_feature_inner[i];
    if (f < d.nfn) ++col_splits_[d.meta_host[f].hist_off >> 8];
  }
  std::vector<int> cand;
  for (int c = 0; c < static_cast<int>(col_splits_.size()); ++c)
    if (col_splits_[c] > 0 && col_slot_host_[c] < 0) cand.push_back(c);
  std::stable_sort(cand.begin(), cand.end(), [&](int a, int b) { return col_splits_[a] > col_splits_[b]; });
  ColumnJobs jobs{};
  for (int c : cand) {
    if (jobs.n == kColumnBuildsMax) break;
    int slot = -1, victim = -1;
    for (int s = 0; s < static_cast<int>(slot_col_.size()) && slot < 0; ++s) {
      const int held = slot_col_[s];
      if (held < 0) slot = s;
      else if (victim < 0 || col_splits_[held] < col_splits_[slot_col_[victim]]) victim = s;
    }
    if (slot < 0) {
      if (col_splits_[slot_col_[victim]] >= col_splits_[c]) break;      // candidates come in descending order: none later wins either
      slot = victim;
      col_slot_host_[slot_col_[slot]] = -1;
      ++cache_evictions_;
    }
    slot_col_[slot] = c;
    col_slot_host_[c] = slot;
    jobs.col[jobs.n] = c; jobs.slot[jobs.n] = slot; ++jobs.n;
  }
  if (jobs.n == 0) return;
  const long long words = (static_cast<long long>(d.num_data) + 3) / 4;
  const unsigned gx = static_cast<unsigned>(std::max<long long>(1, std::min<long long>((words + 255) / 256, static_cast<long long>(num_sms_) * 8)));
  k_tiles_to_column_slots<<<dim3(gx, jobs.n), 256, 0, stream_>>>(d.bins.p, d.rows_stride, d.num_data, jobs, bins_cols_.p, cols_stride_);
  B200_CUDA(cudaGetLastError());
  col_slot_.Upload(col_slot_host_.data(), col_slot_host_.size(), stream_);
  cache_builds_ += jobs.n;
  timing_.launches += 1;
}

void TreeLearner::GetColumnCacheInfo(int64_t* out4) const {
  out4[0] = static_cast<int64_t>(slot_col_.size());
  out4[1] = static_cast<int64_t>(std::count_if(slot_col_.begin(), slot_col_.end(), [](int c) { return c >= 0; }));
  out4[2] = cache_builds_;
  out4[3] = cache_evictions_;
}

void TreeLearner::LaunchPartition(int grid, int last) {
  const Dataset& d = train_;
  TreeCtrl* ctrl = ctrl_.p;
  LeafState* leaves = leaves_.p;
  TreeDev tree = tree_dev_;
  uint8_t* flags = flags_.p;
  const FeatMeta* meta = d.meta.p;
  SplitParams sp = sp_;
  const uint8_t* bins = d.bins.p;
  size_t rows_stride = d.rows_stride;
  int* i0 = idx0_.p; int* i1 = idx1_.p;
  unsigned* bits = part_bits_.p;
  int* chunks = part_chunks_.p;
  const int4* qgh = qgh_.p;
  int4* qord = qord_.p;
  long long* H = H_.p;
  size_t h_elems = slot_elems_;
  const uint16_t* bins16 = d.bins16.p;
  int tickets_per_block = kPartTickets;
  const uint8_t* cols = bins_cols_.p;
  size_t cols_stride = cols_stride_;
  const int* col_slot = col_slot_.p;
  int* super_tot = part_chunks_.p + (d.num_data / kPartChunk + 2);
  const int* bundle_base = d.BundleBase();
  void* args[] = {&ctrl, &leaves, &tree, &flags, &meta, &sp, &last, &bins, &rows_stride, &i0, &i1, &bits, &chunks, &qgh, &qord, &H, &h_elems, &bins16, &tickets_per_block,
                  &cols, &cols_stride, &col_slot, &super_tot, &bundle_base};
  B200_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(k_partition), dim3(grid), dim3(256), args, 0, stream_));
}

// One tree: the whole leaf-wise growth is enqueued without a host sync; leaf choice, smaller/larger
// selection, partition sizes all live in TreeCtrl / LeafState on the device.
void TreeLearner::Grow(const float* g, const float* h, bool const_hessian, const Bag* bag, int tree_index) {
  EnsureColumnCopy();
  const Dataset& d = train_;
  const int n = d.num_data;
  const int L = cfg_.num_leaves;
  rows_ = bag ? bag->count : n;
  TreeCtrl* ctrl = ctrl_.p;
  cudaStream_t s = stream_;
  const int egrid = num_sms_ * 8;
  nvtxRangePushA("b200gbm:K3 quantize + C1 root sums");
  B200_CUDA(cudaMemsetAsync(&ctrl->absmax_bits[0], 0, 8, s));
  k_absmax<<<egrid, 256, 0, s>>>(g, h, n, ctrl);
  if (parallel_) Net().AllReduce(&ctrl->absmax_bits[0], 2, ncclUint32, ncclMax, s);
  k_set_scale<<<1, 1, 0, s>>>(ctrl, const_hessian ? 1 : 0, 1.0);
  // quantised training: B = num_grad_quant_bins levels instead of the 36-bit grid, and K4's packed plane below
  const int quant_bins = cfg_.use_quantized_grad ? cfg_.num_grad_quant_bins : 0;
  if (quant_bins > 0) {
    k_set_quant_scale<<<1, 1, 0, s>>>(ctrl, const_hessian ? 1 : 0, quant_bins);
    k_quantize_discrete<<<egrid, 256, 0, s>>>(g, h, n, qgh_.p, ctrl, const_hessian ? 1 : 0, bag ? bag->in_bag : nullptr, rows_, quant_bins,
                                              cfg_.stochastic_rounding ? 1 : 0, cfg_.data_random_seed, tree_index);
    timing_.launches += 1;
  } else {
    k_quantize<<<egrid, 256, 0, s>>>(g, h, n, qgh_.p, ctrl, const_hessian ? 1 : 0, bag ? bag->in_bag : nullptr, rows_);
  }
  if (parallel_) Net().AllReduce(&ctrl->root_q[0], 3, ncclInt64, ncclSum, s);
  ResetFeaturesByTree();
  if (bag)      // the root leaf is the ascending in-bag row list (SetBaggingData); partitions then ping-pong idx0/idx1 as usual
    B200_CUDA(cudaMemcpyAsync(idx0_.p, bag->rows, static_cast<size_t>(bag->count) * sizeof(int), cudaMemcpyDeviceToDevice, s));
  // the ColSampler stream passes to the device after the tree's feature_fraction draw (ReadTree takes it back)
  k_tree_init<<<1, 256, 0, s>>>(ctrl, leaves_.p, tree_dev_, flags_.p, sp_, rows_, feature_used_.p, bag ? 1 : 0, col_rand_.state());
  nvtxRangePop();
  timing_.launches += 4;
  // forced splits: the plan's evaluations start as "not evaluated" (gain 0) in every tree
  const ForcedArgs forced = forced_host_.empty() ? ForcedArgs{} : ForcedArgs{forced_.p, forced_evals_.p, static_cast<int>(forced_host_.size())};
  if (forced.nodes) forced_evals_.Zero(s);
  const int pgrid = std::max(1, std::min(n / kPartChunk + 1, part_max_blocks_));
  // one block per (leaf, tile feature); the pick step in the last block also sees the wide features' candidates.  Per-node feature
  // sampling adds one column: each leaf's d_bynode_sample block
  const dim3 sgrid(std::max(1, d.nfn) + (bynode_ ? 1 : 0), 2);
  const RowBlockBound bound = d.BlockBound();
  SplitParams sp_local = sp_;      // voting: the local scan's config ([UPSTREAM] VotingParallelTreeLearner::Init local_config_)
  if (voting_) { sp_local.min_data_in_leaf /= Net().world; sp_local.min_sum_hessian /= Net().world; }
  // B200GBM_SPLIT_TIMING=1 (debug): an event after every operation of a split; per-operation averages go to stderr when the learner is freed
  static const bool split_timing = getenv("B200GBM_SPLIT_TIMING") != nullptr;
  auto mark = [&]() { if (split_timing) { cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, s); split_events_.push_back(e); } };
  // round 0's controller is its own launch; every later round's runs in the tail of the previous round's partition kernel
  k_round_ctl<<<1, 256, 0, s>>>(ctrl, leaves_.p, tree_dev_, flags_.p, d.meta.p, sp_, 0);
  timing_.launches += 1;
  for (int split = 0; split < L - 1; ++split) {
    mark();
    if (profile_hist) { cudaEvent_t a, b; B200_CUDA(cudaEventCreate(&a)); B200_CUDA(cudaEventCreate(&b)); hist_events_.push_back(a); hist_events_.push_back(b); B200_CUDA(cudaEventRecord(a, s)); }
    // leaf order of the (g,h) words: written by the previous split's partition kernel; only a bagged root needs its own pass
    if (split == 0 && bag) k_gather_q<<<egrid, 256, 0, s>>>(&ctrl->hist_work, idx0_.p, idx1_.p, qgh_.p, qord_.p);
    mark();
    // the scratch histogram H is zero here: zeroed at set-up and by every partition kernel after the scan consumed it
    nvtxRangePushA("b200gbm:K4 histogram");
    launch_k4(const_hessian, quant_bins, d.bins.p, d.rows_stride, d.num_tiles, qgh_.p, qord_.p, idx0_.p, idx1_.p, &ctrl->hist_work,
              reinterpret_cast<unsigned long long*>(H_.p), bound, num_sms_, s);
    if (d.nw > 0) {      // the features with more than 256 bins: own sub-histogram layout (k4_hist_wide)
      int max_nb = 0, units = 0;
      for (int u = d.nfn; u < d.nf; ++u) {
        max_nb = std::max(max_nb, d.meta_host[u].num_bin);
        units += (d.meta_host[u].num_bin + kWideHistSeg - 1) / kWideHistSeg;
      }
      const int segs = (max_nb + kWideHistSeg - 1) / kWideHistSeg;      // z: 8192-bin segments of the largest feature
      // x: row parts, chosen so that the CTAs that have work (a (feature, segment) pair past the feature's last bin exits at once) make
      // about four waves of one CTA per SM (128 KB of shared memory each)
      const dim3 wgrid(static_cast<unsigned>(std::max(1, std::min(64, 4 * num_sms_ / std::max(1, units)))), static_cast<unsigned>(d.nw), static_cast<unsigned>(segs));
      if (const_hessian)
        k4_hist_wide<3><<<wgrid, kWideThreads, 4 * kWideHistSeg * 4, s>>>(d.bins16.p, d.rows_stride, d.meta.p + d.nfn, qgh_.p, qord_.p, idx0_.p, idx1_.p, &ctrl->hist_work,
                                                                         reinterpret_cast<unsigned long long*>(H_.p));
      else
        k4_hist_wide<4><<<wgrid, kWideThreads, 4 * kWideHistSeg * 4, s>>>(d.bins16.p, d.rows_stride, d.meta.p + d.nfn, qgh_.p, qord_.p, idx0_.p, idx1_.p, &ctrl->hist_work,
                                                                         reinterpret_cast<unsigned long long*>(H_.p));
      timing_.launches += 1;
    }
    nvtxRangePop();
    if (profile_hist) B200_CUDA(cudaEventRecord(hist_events_.back(), s));
    mark();
    // the dynamic scratch of k_scan is only touched by categorical features and bundle members
    const int scan_smem = (d.has_categorical || !d.bundles.empty()) ? kScanSmem : 0;
    // every scan gets the device constraint arrays, so no instantiation can read through a null pointer
    const ConstraintArgs cons{mono_.p, monotone_penalty_, sets_of_.p};
    if (voting_) {
      // local scan + top-k -> all-gather of the records -> vote + pack -> all-reduce of the packed columns -> global scan + pick
      nvtxRangePushA("b200gbm:voting local scan + vote + C2 reduce + global scan + pick");
      const VoteBufs vote{recs_.p, voted_.p, packed_.p, top_k_};
      k_scan<kScanLocal><<<sgrid, 256, scan_smem, s>>>(ctrl, leaves_.p, d.meta.p, H_.p, pool_.p, slot_elems_, flags_.p, cands_.p, sp_local, d.BundleBase(), vote, xrand_.p,
                                                        cons, NodeSampleArgs{}, ForcedArgs{});
      mark();
      Net().AllGather(recs_.p, all_recs_.p, recs_.n * sizeof(VoteRec), s);
      mark();
      const int R = Net().world;
      k_vote_pack<<<2 * top_k_, 256, static_cast<size_t>(R) * top_k_ * (sizeof(double) + sizeof(int)), s>>>(
          ctrl, leaves_.p, d.meta.p, d.BundleBase(), all_recs_.p, R, top_k_, H_.p, pool_.p, slot_elems_, voted_.p, packed_.p);
      mark();
      Net().AllReduce(packed_.p, packed_.n, ncclInt64, ncclSum, s);
      mark();
      k_scan<kScanGlobal><<<sgrid, 256, scan_smem, s>>>(ctrl, leaves_.p, d.meta.p, H_.p, pool_.p, slot_elems_, flags_.p, cands_.p, sp_, d.BundleBase(), vote, xrand_.p,
                                                         cons, NodeSampleArgs{}, ForcedArgs{});
      nvtxRangePop();
      comm_hist_bytes_ += static_cast<long long>(packed_.n * sizeof(long long));
      comm_rec_bytes_ += static_cast<long long>(all_recs_.n * sizeof(VoteRec));
      timing_.launches += 2;
    } else {
      nvtxRangePushA(parallel_ ? "b200gbm:C2 histogram reduce + K5 scan + pick" : "b200gbm:K5 scan + pick");
      if (parallel_) {
        Net().AllReduce(H_.p, slot_elems_, ncclInt64, ncclSum, s);   // C2
        comm_hist_bytes_ += static_cast<long long>(slot_elems_ * sizeof(long long));
      }
      mark();
      const ScanKernels& k = kScanKernels[extra_trees_][monotone_ || smooth_];
      if (d.nw > 0) {
        k.scan_wide<<<dim3(d.nw, 2), 256, kWideMaxBins * 8, s>>>(ctrl, leaves_.p, d.meta.p, H_.p, pool_.p, slot_elems_, flags_.p, cands_.p, sp_, xrand_.p,
                                                                 cons, forced);
        timing_.launches += 1;
      }
      // scan + (last block) pick
      const NodeSampleArgs node = bynode_ ? NodeSampleArgs{node_mask_.p, node_work_.p, real_order_.p, feature_used_.p, bynode_k_} : NodeSampleArgs{};
      k.scan<<<sgrid, 256, scan_smem, s>>>(ctrl, leaves_.p, d.meta.p, H_.p, pool_.p, slot_elems_, flags_.p, cands_.p, sp_, d.BundleBase(), VoteBufs{}, xrand_.p,
                                           cons, node, forced);
      nvtxRangePop();
    }
    mark();
    comm_splits_ += 1;
    nvtxRangePushA("b200gbm:K7 partition + controller");
    LaunchPartition(pgrid, split == L - 2 ? 1 : 0);
    nvtxRangePop();
    mark();
    timing_.launches += 3; timing_.hist_launches += 1;
  }
}

void TreeLearner::AddScore(double* score_k, double shrinkage) {
  k_add_score<<<num_sms_ * 8, 256, 0, stream_>>>(ctrl_.p, leaves_.p, tree_dev_, idx0_.p, idx1_.p, score_k, shrinkage);
}

void TreeLearner::ReadTree(HostTree* out) {
  const Dataset& d = train_;
  cudaStream_t s = stream_;
  B200_CUDA(cudaMemcpyAsync(tree_host_, tree_blob_.p, tree_blob_.n, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaMemcpyAsync(ctrl_host_, ctrl_.p, sizeof(TreeCtrl), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  if (!split_events_.empty()) {
    static const char* kOps[] = {"gather_q(bagged root)", "K4", "allreduce", "scan+pick", "partition+zeroH+ctl"};
    static const char* kVotingOps[] = {"gather_q(bagged root)", "K4", "local scan+top-k", "allgather", "vote+pack", "allreduce", "global scan+pick",
                                       "partition+zeroH+ctl"};
    const char* const* ops = voting_ ? kVotingOps : kOps;
    const int per = voting_ ? 9 : 6;       // marks per split
    for (size_t b0 = 0; b0 + per <= split_events_.size(); b0 += per)
      for (int o = 0; o < per - 1; ++o) { float ms = 0; cudaEventElapsedTime(&ms, split_events_[b0 + o], split_events_[b0 + o + 1]); split_op_ms_[ops[o]] += ms; }
    split_op_trees_ += 1;
    for (auto e : split_events_) cudaEventDestroy(e);
    split_events_.clear();
  }
  if (!hist_events_.empty()) {
    for (size_t i = 0; i + 1 < hist_events_.size(); i += 2) { float ms = 0; cudaEventElapsedTime(&ms, hist_events_[i], hist_events_[i + 1]); timing_.hist_ms += ms; }
    for (auto e : hist_events_) cudaEventDestroy(e);
    hist_events_.clear();
  }
  timing_.hist_rows += ctrl_host_->trace_rows;
  col_rand_.set_state(ctrl_host_->col_state);      // the ColSampler stream after the tree's per-node draws (none without them)
  // ---- host copy of the tree
  const TreeDev t = TreeAt(tree_host_);
  const int nl = *t.num_leaves;
  out->Resize(nl);
  if (nl > 1) {
    for (int i = 0; i < nl - 1; ++i) {
      const int sf = t.split_feature_inner[i], tb = t.threshold_bin[i], dt = t.decision_type[i];
      out->left_child[i] = t.left_child[i]; out->right_child[i] = t.right_child[i]; out->split_feature_inner[i] = sf;
      out->split_feature[i] = d.used[sf]; out->threshold_in_bin[i] = static_cast<uint32_t>(tb);
      out->decision_type[i] = static_cast<int8_t>(dt); out->split_gain[i] = t.split_gain[i];
      const FeatureBins& fbm = d.mappers[d.used[sf]];
      if (dt & 1) {          // categorical node: bins of the inner bitset -> category values ([UPSTREAM] RealThreshold per bin)
        std::vector<int> cats;
        if (sf >= d.nfn) { for (int k = 0; k < t.cat_list_len[i]; ++k) cats.push_back(fbm.bin_to_cat[t.cat_list[i * kCatListMax + k]]); }
        else for (int b = 0; b < fbm.num_bin; ++b) if ((t.cat_bits[i * 8 + (b >> 5)] >> (b & 31)) & 1u) cats.push_back(fbm.bin_to_cat[b]);
        out->AddCategoricalNode(i, cats);
      } else {
        double thr = fbm.upper[tb];
        if (std::isnan(thr)) thr = 0.0; else if (thr >= 1e300) thr = 1e300; else if (thr <= -1e300) thr = -1e300;
        out->threshold[i] = thr;
      }
      out->internal_value[i] = t.internal_value[i]; out->internal_weight[i] = t.internal_weight[i]; out->internal_count[i] = t.internal_count[i];
    }
    for (int i = 0; i < nl; ++i) { out->leaf_value[i] = t.leaf_value[i]; out->leaf_weight[i] = t.leaf_weight[i]; out->leaf_count[i] = t.leaf_count[i]; out->leaf_depth[i] = t.leaf_depth[i]; }
  } else {
    out->leaf_value[0] = 0.0;
  }
  UpdateColumnCache(*out);
}

}  // namespace b200gbm
