// sm_90a kernels of the b200gbm training engine other than K4 (hist_kernel.cuh).
// Kernel numbering follows SURVEY.md §2.5.  Everything a tree needs lives in device memory
// (leaf table, control block, tree arrays) so the host enqueues a whole tree without a sync.
#pragma once
#include <climits>
#include <cstdint>
#include <cuda_runtime.h>
#include "config.h"
#include "hist_kernel.cuh"

namespace b200gbm {

constexpr double kEpsD = 1e-15;
#define kNegInf (-__longlong_as_double(0x7ff0000000000000LL))   /* -inf, usable in device code */

struct FeatMeta {          // per inner (used) feature
  int num_bin;
  int missing_type;        // 0 none, 2 NaN
  int default_bin;
  int offset;              // 1 iff most_freq_bin == 0  ([UPSTREAM] storage convention, affects NaN forward scan)
  int real_index;
  int is_categorical;      // bins are category ranks; splits are bin bitsets
  int num_sorted_cats;     // categorical: entries of the sorted category table (ub row = categories, catbin row = their bins)
  int hist_off;            // first (g,h) pair of the feature's storage column in a histogram slot: col * 256 for a tile feature (col = u
                           // without feature bundles), beyond the tiles for a wide one
  int table_off;           // first entry of the feature's row in the bin tables ub / catbin: u * 256 for a tile feature, beyond the
                           // tile rows for a wide one
};

// Exclusive feature bundles (bundle.h): a bundle column holds several features of which at most one is away from its most frequent bin
// (mfb = default_bin for a member) in any row.  Slot 0 = every member at its mfb; member bin b != mfb is stored at
// base + 1 + (b < mfb ? b : b - 1).  Decoding a stored slot back to the member's bin:
__host__ __device__ __forceinline__ unsigned d_unbundle(unsigned slot, int base, int mfb, int num_bin) {
  if (base < 0) return slot;
  const int v = static_cast<int>(slot) - base - 1;
  if (v < 0 || v >= num_bin - 1) return static_cast<unsigned>(mfb);
  return static_cast<unsigned>(v < mfb ? v : v + 1);
}
// slot of member bin `bin` (the caller has checked bin != mfb)
__host__ __device__ __forceinline__ unsigned d_bundle_slot(unsigned bin, int base, int mfb) {
  return static_cast<unsigned>(base + 1) + (bin < static_cast<unsigned>(mfb) ? bin : bin - 1);
}

// "Wide" features: more than 256 bins.  LightGBM does not cap a categorical feature at max_bin — it keeps categories until 99 % of the
// sampled mass is covered (BinMapper::FindBin) — so a 10^3..10^5-cardinality column (BASELINE.json configs[4]) needs thousands of bins.
// They live outside the uint8 feature tiles: one uint16 column per feature, their own histogram kernel (k4_hist_wide) and scan
// (k_scan_wide); inner index = nfn + w, described by meta[nfn + w] like every other feature.  A categorical split on one sends at most
// max_cat_threshold bins left, carried as a bin list.
constexpr int kWideHistSeg = 8192;       // bins one k4_hist_wide CTA accumulates: 4 planes x 8192 x 4 B = 128 KB of shared memory
constexpr int kWideMaxBins = 16384;      // per feature (k_scan_wide sorts (ctr, bin) keys in 160 KB of shared memory); more fails loudly
constexpr int kCatListMax = 64;          // >= max_cat_threshold (default 32) when wide features exist
struct BinView {                         // where a row's bin of inner feature u is stored
  const uint8_t* bins; size_t rows_stride; const uint16_t* bins16; int nfn;
  const FeatMeta* meta; const int* bundle_base;      // bundle_base null: no feature bundle, column = feature, no decode
  __device__ __forceinline__ unsigned at(int u, size_t row) const {
    if (u >= nfn) return bins16[static_cast<size_t>(u - nfn) * rows_stride + row];
    if (!bundle_base) return bins[(static_cast<size_t>(u >> 5) * rows_stride + row) * 32 + (u & 31)];
    const int c = meta[u].hist_off >> 8;
    return d_unbundle(bins[(static_cast<size_t>(c >> 5) * rows_stride + row) * 32 + (c & 31)], bundle_base[u], meta[u].default_bin, meta[u].num_bin);
  }
};

struct SplitParams {
  double l1, l2, max_delta_step, min_gain_to_split, min_sum_hessian;
  int min_data_in_leaf, max_depth, num_leaves, parallel;
  int nf, nf_pad, num_tiles, nfn;                              // nfn: features stored in uint8 tiles; [nfn, nf) are wide
  double cat_l2, cat_smooth;                                   // categorical split search ([UPSTREAM] defaults 10, 10)
  int max_cat_threshold, max_cat_to_onehot, min_data_per_group;         // 32, 4, 100
  int interaction;                                             // 1 when interaction_constraints is non-empty (d_pick_block, d_round_ctl)
  double path_smooth;                                          // > kPathSmoothEps: outputs and gains smoothed (d_smooth_output)
};

// extra_trees (the scans' template parameter kExtra; [UPSTREAM] FeatureHistogram USE_RAND, FeatureMetainfo::rand): every used feature
// owns one LCG, seeded extra_seed + i with i the feature's position among the used features in real-index order.  Each scan of the
// feature in a leaf whose draw range is non-empty takes one draw, the smaller leaf's before the larger's: NextInt(0, range) = (x & 0x7fffffff) % range after x = 214013 x + 2531011.
// An empty range draws nothing and leaves the threshold at 0, as upstream does.  The stream states live in xrand[0, nf_pad); the
// scan block of (leaf `which`, feature u) writes its number of draws (0 or 1) to xrand[(1 + which) * nf_pad + u], and the block that runs
// the pick step advances the states by them once every scan block of the round has finished (d_extra_commit).
__host__ __device__ __forceinline__ unsigned d_lcg_next(unsigned x) { return 214013u * x + 2531011u; }
__device__ __forceinline__ int d_extra_draw(unsigned* x, int range) {
  if (range <= 0) return 0;
  *x = d_lcg_next(*x);
  return static_cast<int>((*x & 0x7fffffffu) % static_cast<unsigned>(range));
}
// seeds every feature's stream: xrand[u] = extra_seed + pos[u], pos[u] = the feature's position among the used features in real-index order
__global__ void k_extra_seed(unsigned* __restrict__ xrand, const int* __restrict__ pos, int nf, int extra_seed) {
  for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < nf; u += gridDim.x * blockDim.x) xrand[u] = static_cast<unsigned>(extra_seed + pos[u]);
}
// many-vs-many categorical search: the draw range given the number of bins with >= cat_smooth rebuilt rows
// (max(min(max_num_cat, used_bin) - 1, 0) with max_num_cat = min(max_cat_threshold, (used_bin + 1) / 2))
__device__ __forceinline__ int d_cat_rand_range(int used_bin, int max_cat_threshold) {
  const int max_num_cat = min(max_cat_threshold, (used_bin + 1) / 2);
  return max(min(max_num_cat, used_bin) - 1, 0);
}

struct SplitCand {         // best threshold of one (leaf, feature)
  double gain;             // best_gain - min_gain_shift, or -inf
  double left_g, left_h;   // best_sum_left_gradient / _hessian (hessian still carries +kEpsilon)
  int threshold, left_count, default_left, feature;   // feature = inner index
  double l2_extra;         // cat_l2 for a many-vs-many categorical split (leaf outputs use lambda_l2 + l2_extra)
  unsigned cat_bits[8];    // categorical: bins that go LEFT
  int is_cat, cat_list_len;
  unsigned short cat_list[kCatListMax];      // wide categorical feature: the bins that go LEFT (cat_bits unused)
};

struct LeafBest {
  double gain;
  double left_g, left_h, right_g, right_h;   // sums as stored in SplitInfo (epsilon removed)
  double left_out, right_out;
  int feature, threshold, default_left, left_count, right_count, is_cat;
  unsigned cat_bits[8];
  int cat_list_len, monotone_type;           // monotone_type: the split feature's constraint (0 without monotone constraints)
  unsigned short cat_list[kCatListMax];
  unsigned long long inter_sets;             // interaction constraints: the split feature's sets_of word (0 without them)
};

struct LeafState {
  int begin, count, buf, depth;
  int global_count, identity, hist_slot, parent_node;
  double sum_g, sum_h;
  LeafBest best;
  // exact fixed-point (g,h) totals, kept only for datasets with feature bundles: qtot = this leaf's (written by k_scan), qpar = its
  // parent's (written by the round controller); a bundle member's most frequent bin is the leaf total minus its other bins
  long long qtot[2], qpar[2];
  // monotone constraints (basic method): the bounds [mono_min, mono_max] of this leaf's output; the root's are (-inf, +inf), children
  // inherit their parent's and a numerical split on a monotone feature narrows them at the mid-point of the two outputs (d_round_ctl)
  double mono_min, mono_max;
  // path smoothing: this leaf's output, the parent_output its scans smooth toward ([UPSTREAM] LeafSplits::weight).  A child's is the
  // smoothed (and clamped) output the pick step gave it; the root's is its own unsmoothed output (k_tree_init).
  double output;
  // interaction constraints: bit s is set when constraint set s holds every split feature on the path from the root to this leaf.  The
  // root's has every bit; a split on feature u gives both children parent & sets_of[u] (d_round_ctl).  Read only when p.interaction.
  unsigned long long inter_mask;
};

// The scans' constraint arguments.
// Monotone constraints ([UPSTREAM] monotone_constraints.hpp BasicLeafConstraints, FeatureHistogram USE_MC): the scans' template parameter
// kMono, which path smoothing (USE_SMOOTHING) turns on too.  type: per inner feature -1, 0 or +1 (the real feature's
// monotone_constraints entry, all 0 without a list); penalty: monotone_penalty.
// Interaction constraints ([UPSTREAM] ColSampler::GetByNode): sets_of[u], per inner feature, has bit s set when constraint set s holds
// the feature's real index; feature u may split a leaf iff sets_of[u] & inter_mask != 0.  Read by the pick step only when p.interaction.
struct ConstraintArgs { const signed char* type; double penalty; const unsigned long long* sets_of; };
// Per-node feature sampling ([UPSTREAM] ColSampler::GetByNode with feature_fraction_bynode < 1), k_scan's argument: d_bynode_sample
// writes mask[which][u] = 1 for the features the leaf of the round samples, and the pick step passes over the others.  mask is null
// without per-node sampling (nothing is read then).  k = GetCnt(|tree sample|, feature_fraction_bynode); order: the used features in
// real-index order (Dataset::sample_order); tree_used: the tree's feature_fraction sample; work: [2][4][nf_pad] ints of scratch.
struct NodeSampleArgs { uint8_t* mask; int* work; const int* order; const uint8_t* tree_used; int k; };
// Forced splits ([UPSTREAM] SerialTreeLearner::ForceSplits; forced_splits.h builds the plan): the plan's nodes in breadth-first order.
// Node j is the j-th split of the tree while the forced phase lasts, so it splits leaf `leaf` (the root's is 0, a left child keeps its
// parent's leaf, a right child of node j gets leaf j + 1).  bin: the threshold's bin (numerical) or the category's bin (categorical, 0
// when the category has no bin of its own); left / right: the child plan nodes, -1 for none.  A node is evaluated by the scan block of
// (its leaf, its feature) in the round that scans its leaf (d_forced_eval) into evals[node]; the evals are zeroed before each tree, so
// a gain that is not > 0 is a node that was never evaluated or is invalid.  nodes null: no plan, and nothing else is read.
struct ForcedNode { int feature, bin, is_cat, leaf, left, right; };
struct ForcedArgs { const ForcedNode* nodes; SplitCand* evals; int n; };

struct TreeCtrl {
  int num_leaves, left_leaf, right_leaf, smaller, larger, go, finished, split_leaf;
  int split_feature, split_threshold, split_default_left, split_missing_type, split_num_bin, new_leaf, pending, pad;
  int part_begin, part_count, part_buf, part_identity, part_left_total, smaller_rows, round, split_is_cat;
  unsigned split_cat_bits[8];
  HistWork hist_work;
  unsigned absmax_bits[2];     // max|g|, max|h| as float bits (non-negative floats order like uints)
  int exp_g, exp_h;            // fixed-point exponents: q = rint(x * 2^exp)
  double inv_g, inv_h;         // hist value -> real value
  long long root_q[4];         // sum q_g, sum q_h, local rows, unused  (allreduced)
  long long trace_rows;        // sum of rows scanned by K4 this tree (for the roofline byte model)
  unsigned scan_ticket;        // blocks of k_scan that finished this round (the last one runs the pick step)
  int q_side;                  // (unused since the fused partition kernel decides the side itself)
  unsigned part_barrier;       // k_partition: grid-barrier arrive counter (reset by its last block)
  unsigned part_ticket;        // k_partition: finished-block ticket (the last block runs the next round's controller)
  unsigned part_next[2];       // k_partition: next chunk of phase 1 / phase 3 (dynamic hand-out; reset by its last block)
  int split_wide;              // wide index (inner feature - nfn) of the split feature, or -1
  int split_cat_list_len;
  unsigned short split_cat_list[kCatListMax];
  // per-node feature sampling: the ColSampler stream's state.  k_tree_init takes it from the host after the tree's feature_fraction
  // draw, the pick step advances it to col_next (written by d_bynode_sample) each round, and ReadTree hands it back to the host.
  unsigned col_state, col_next;
  // forced splits: the plan node the next forced split applies, -1 once the forced phase is over (k_tree_init starts it at 0; read only
  // with a plan)
  int forced_next;
};

struct TreeDev {               // SoA tree under construction (sizes: num_leaves / num_leaves-1)
  int* left_child; int* right_child; int* split_feature_inner; int* threshold_bin; int* decision_type;
  float* split_gain; double* leaf_value; double* leaf_weight; int* leaf_count; double* internal_value;
  double* internal_weight; int* internal_count; int* leaf_parent; int* leaf_depth; int* num_leaves;
  unsigned* cat_bits;          // [num_leaves-1][8] inner (bin) bitset of categorical nodes
  unsigned short* cat_list;    // [num_leaves-1][kCatListMax] bins going left at a categorical node on a wide feature
  int* cat_list_len;           // [num_leaves-1] 0 for every other node
};

// ---------------------------------------------------------------- helpers
__device__ __forceinline__ double d_sign(double x) { return (x > 0.0) - (x < 0.0); }
__device__ __forceinline__ double d_threshold_l1(double s, double l1) {
  double r = fmax(0.0, fabs(s) - l1);
  return d_sign(s) * r;
}
__device__ __forceinline__ double d_calc_output(double g, double h, const SplitParams& p) {
  double ret = (p.l1 > 0) ? -d_threshold_l1(g, p.l1) / (h + p.l2) : -g / (h + p.l2);
  if (p.max_delta_step > 0 && fabs(ret) > p.max_delta_step) ret = d_sign(ret) * p.max_delta_step;
  return ret;
}
// NOT inlined on purpose: the split scan evaluates it ~40 times per lane; inlined and unrolled (each call holds a software fp64 division)
// k_scan grew to 15.8K SASS instructions that every warp ran through once, and ncu showed 55 % of its stall samples in stall_no_inst
// (instruction-cache misses), 39 us per launch.  As a function its body is fetched once.
__device__ __noinline__ double d_leaf_gain(double g, double h, const SplitParams& p) {
  if (!(p.max_delta_step > 0)) {
    if (p.l1 > 0) { double sg = d_threshold_l1(g, p.l1); return (sg * sg) / (h + p.l2); }
    return (g * g) / (h + p.l2);
  }
  double out = d_calc_output(g, h, p);
  double sg = (p.l1 > 0) ? d_threshold_l1(g, p.l1) : g;
  return -(2.0 * sg * out + (h + p.l2) * out * out);
}
// path smoothing ([UPSTREAM] CalculateSplittedLeafOutput<USE_SMOOTHING>): the output of a leaf of n rows (L1, l2, max_delta_step as
// d_calc_output), then, when p.path_smooth > kPathSmoothEps, ret * (n/s) / (n/s + 1) + parent_output / (n/s + 1) in that order.
// Out of line for d_leaf_gain's reason.
__device__ __noinline__ double d_smooth_output(double g, double h, int n, double parent_output, const SplitParams& p) {
  double ret = d_calc_output(g, h, p);
  if (p.path_smooth > kPathSmoothEps) {
    const double w = n / p.path_smooth;
    ret = ret * w / (w + 1) + parent_output / (w + 1);
  }
  return ret;
}
// path smoothing: a leaf's gain at its smoothed output ([UPSTREAM] GetLeafGain<USE_SMOOTHING>, never clamped to monotone bounds), the
// scans' min_gain_shift; d_leaf_gain's when smoothing is off.  Out of line for d_leaf_gain's reason.
__device__ __noinline__ double d_smooth_leaf_gain(double g, double h, int n, double parent_output, const SplitParams& p) {
  if (!(p.path_smooth > kPathSmoothEps)) return d_leaf_gain(g, h, p);
  const double out = d_smooth_output(g, h, n, parent_output, p);
  const double sg = (p.l1 > 0) ? d_threshold_l1(g, p.l1) : g;
  return -(2.0 * sg * out + (h + p.l2) * out * out);
}
// monotone constraints: a child's output of n rows, CalculateSplittedLeafOutput (smoothed toward parent_output when path smoothing is
// on) clamped to the leaf's bounds
__device__ __forceinline__ double d_mono_output(double g, double h, int n, double parent_output, const SplitParams& p, double lo, double hi) {
  double ret = d_smooth_output(g, h, n, parent_output, p);
  if (ret < lo) ret = lo;
  else if (ret > hi) ret = hi;
  return ret;
}
// The kMono scans' split gain ([UPSTREAM] GetSplitGains<USE_MC, USE_SMOOTHING>): both children's outputs (of lc and rc rows, smoothed
// toward the leaf's output `parent_output` when path smoothing is on) clamped to the leaf's bounds [lo, hi], then
// GetLeafGainGivenOutput(left) + GetLeafGainGivenOutput(right) = -(2 ThresholdL1(g) out + (h + l2) out^2) at those outputs; 0 when the
// outputs break the split feature's direction `mono` (left > right for +1, left < right for -1).  Without monotone constraints the
// bounds are (-inf, +inf) and mono is 0, which leaves the smoothed gain.  Out of line for d_leaf_gain's reason.
__device__ __noinline__ double d_mono_split_gain(double lg, double lh, double rg, double rh, int lc, int rc, double parent_output, const SplitParams& p,
                                                 double lo, double hi, int mono) {
  const double lo_out = d_mono_output(lg, lh, lc, parent_output, p, lo, hi), ro_out = d_mono_output(rg, rh, rc, parent_output, p, lo, hi);
  if ((mono > 0 && lo_out > ro_out) || (mono < 0 && lo_out < ro_out)) return 0.0;
  const double slg = (p.l1 > 0) ? d_threshold_l1(lg, p.l1) : lg, srg = (p.l1 > 0) ? d_threshold_l1(rg, p.l1) : rg;
  return -(2.0 * slg * lo_out + (lh + p.l2) * lo_out * lo_out) + -(2.0 * srg * ro_out + (rh + p.l2) * ro_out * ro_out);
}
// monotone_penalty: the factor on a monotone feature's shifted gain in a leaf of depth d ([UPSTREAM] ComputeMonotoneSplitGainPenalty,
// kEpsilon = 1e-15f)
__device__ __forceinline__ double d_mono_penalty(int depth, double penalty) {
  const double eps = static_cast<double>(1e-15f);
  if (penalty >= depth + 1.0) return eps;
  if (penalty <= 1.0) return 1.0 - penalty / exp2(static_cast<double>(depth)) + eps;
  return 1.0 - exp2(penalty - 1.0 - depth) + eps;
}

// ---------------------------------------------------------------- binning (dataset creation)
// numerical value -> bin (ValueToBin): lower-bound search `value <= ub[m * stride]`
__device__ __forceinline__ unsigned d_num_bin(double v, const FeatMeta& m, const double* ub, int stride) {
  if (isnan(v)) {
    if (m.missing_type == 2) return static_cast<unsigned>(m.num_bin - 1);
    v = 0.0;
  }
  int lo = 0, hi = m.num_bin - 1 - (m.missing_type == 2 ? 1 : 0);
  while (lo < hi) {
    int mid = (hi + lo - 1) / 2;
    if (v <= ub[mid * stride]) hi = mid; else lo = mid + 1;
  }
  return static_cast<unsigned>(lo);
}
// value -> bin of any feature, tile or wide.  row = the feature's ub row (entry i at row[i * stride]), catbin_row = its catbin row.
// Categorical: binary search of the category int(v) in the sorted category values; NaN, negative or unseen -> bin 0.  The values are
// integers stored as doubles, which hold them exactly, so the probes compare doubles and convert nothing.
__device__ __forceinline__ unsigned d_value_to_bin(double v, const FeatMeta& m, const double* row, int stride, const uint16_t* catbin_row) {
  if (!m.is_categorical) return d_num_bin(v, m, row, stride);
  if (isnan(v)) return 0;
  const int iv = static_cast<int>(v);
  if (iv < 0) return 0;
  const double cat = iv;
  int lo = 0, hi = m.num_sorted_cats;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (row[mid * stride] < cat) lo = mid + 1; else hi = mid; }
  return lo < m.num_sorted_cats && row[lo * stride] == cat ? catbin_row[lo] : 0u;
}

// One warp per row-of-a-tile: lane = storage column of the tile.  Upper bounds of the tile's (at most 32) plain features sit
// in shared memory ([32][256] doubles = 64 KB).  col_feat[column] = the plain feature of the column, or -1: a bundle column (left at
// slot 0 here, k_bin_bundles writes its non-default rows) or padding.
template <typename T>
__global__ void __launch_bounds__(256)
k_bin_rows(const T* __restrict__ X, long long nrow, int ncol, int row_major, long long ld, const FeatMeta* __restrict__ meta,
           const double* __restrict__ ub, const uint16_t* __restrict__ catbin, const int* __restrict__ col_feat, uint8_t* __restrict__ bins,
           long long rows_stride, long long row_offset) {
  extern __shared__ double s_ub[];   // [256 bins][32 lanes]: lane l always hits bank pair 2l -> no conflicts beyond the 64-bit 2-phase
  const int tile = blockIdx.y;
  for (int e = threadIdx.x; e < 32 * 256; e += blockDim.x) {
    const int f = col_feat[tile * 32 + (e >> 8)];
    s_ub[(e & 255) * 32 + (e >> 8)] = f >= 0 ? ub[static_cast<size_t>(f) * 256 + (e & 255)] : 0.0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int u = col_feat[tile * 32 + lane];
  FeatMeta m;
  m.num_bin = 1; m.missing_type = 0; m.real_index = 0; m.is_categorical = 0; m.num_sorted_cats = 0;
  if (u >= 0) m = meta[u];
  const double* myub = s_ub + lane;
  for (long long r = blockIdx.x * 8LL + warp; r < nrow; r += gridDim.x * 8LL) {
    unsigned bin = 0;
    if (u >= 0) {
      const double v = row_major ? static_cast<double>(X[r * ld + m.real_index]) : static_cast<double>(X[static_cast<long long>(m.real_index) * ld + r]);
      bin = d_value_to_bin(v, m, myub, 32, catbin + m.table_off);
    }
    bins[(static_cast<size_t>(tile) * rows_stride + row_offset + r) * 32 + lane] = static_cast<uint8_t>(bin);
  }
}

// ---------------------------------------------------------------- exclusive feature bundles (bundle.h): row check and binning
// One member of a bundle; the members of bundle k are [start[k], start[k+1]).  A value is away from the member's most frequent bin
// iff it is NaN and NaN has its own bin, or it lies outside (zlo, zhi] — exactly the values whose bin differs from the mfb.  zlo = -inf
// when the mfb is bin 0, whose range has no lower end (-inf itself lands there).
struct BundleMember {
  double zlo, zhi;
  int real_index, inner, base, bundle;     // inner / base: set once the layout is final (the row check needs neither)
  int nan_moves, pad;
};
__device__ __forceinline__ bool d_off_mfb(double v, const BundleMember& m) {
  return isnan(v) ? m.nan_moves != 0 : !((v > m.zlo || isinf(m.zlo)) && v <= m.zhi);
}
// per bundle: the rows (of this block of rows) in which two or more members are away from their mfb; one thread per (bundle, row)
template <typename T>
__global__ void __launch_bounds__(256)
k_bundle_conflicts(const T* __restrict__ X, long long nrow, int row_major, long long ld, const BundleMember* __restrict__ mem,
                   const int* __restrict__ start, int nb, unsigned long long* __restrict__ conflicts) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < nrow * nb; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(e / nrow);
    const long long r = e - static_cast<long long>(b) * nrow;
    int off = 0;
    for (int k = start[b]; k < start[b + 1]; ++k) {
      const int f = mem[k].real_index;
      const double v = row_major ? static_cast<double>(X[r * ld + f]) : static_cast<double>(X[static_cast<long long>(f) * ld + r]);
      if (d_off_mfb(v, mem[k]) && ++off == 2) { atomicAdd(conflicts + b, 1ull); break; }
    }
  }
}
// CSR: one warp per row.  The bundles that already had a member away from its mfb in this row are listed in shared memory; a second
// one is a conflict.  A row that touches more than kSeenPerWarp bundles counts its further bundles as conflicts (dissolving is always safe).
// conflicts[k] > 0 iff some row has two members of bundle k away from their mfb.
constexpr int kSeenPerWarp = 256;
template <typename TI, typename TV>
__global__ void __launch_bounds__(256)
k_bundle_conflicts_csr(const TI* __restrict__ indptr, const int* __restrict__ indices, const TV* __restrict__ vals, long long nrow, long long elem_base,
                       const int* __restrict__ member_of, const BundleMember* __restrict__ mem, unsigned long long* __restrict__ conflicts) {
  __shared__ int s_seen[8][kSeenPerWarp];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  int* seen_list = s_seen[wib];
  const long long warp = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5, nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long r = warp; r < nrow; r += nwarps) {
    const long long a = static_cast<long long>(indptr[r]) - elem_base, e = static_cast<long long>(indptr[r + 1]) - elem_base;
    int nseen = 0;
    for (long long k0 = a; k0 < e; k0 += 32) {
      const long long k = k0 + lane;
      int bundle = -1;
      if (k < e) {
        const int mi = member_of[indices[k]];
        if (mi >= 0 && d_off_mfb(static_cast<double>(vals[k]), mem[mi])) bundle = mem[mi].bundle;
      }
      const unsigned peers = __match_any_sync(0xffffffffu, bundle);
      const bool leader = bundle >= 0 && __ffs(peers) - 1 == lane;
      bool seen = false;
      if (bundle >= 0) for (int i = 0; i < nseen; ++i) seen |= seen_list[i] == bundle;
      if (leader && (seen || __popc(peers) > 1)) atomicAdd(conflicts + bundle, 1ull);
      const bool add = leader && !seen;
      const unsigned adds = __ballot_sync(0xffffffffu, add);
      __syncwarp();
      if (add) {
        const int pos = nseen + __popc(adds & ((1u << lane) - 1u));
        if (pos < kSeenPerWarp) seen_list[pos] = bundle;
        else atomicAdd(conflicts + bundle, 1ull);
      }
      nseen = min(kSeenPerWarp, nseen + __popc(adds));
      __syncwarp();
    }
  }
}
// the non-default rows of the bundle columns (k_bin_rows left them at slot 0); one thread per (bundle, row).  The row check guarantees
// at most one member per row is away from its mfb.
template <typename T>
__global__ void __launch_bounds__(256)
k_bin_bundles(const T* __restrict__ X, long long nrow, int row_major, long long ld, const BundleMember* __restrict__ mem, const int* __restrict__ start,
              const int* __restrict__ bundle_col, int nb, const FeatMeta* __restrict__ meta, const double* __restrict__ ub, uint8_t* __restrict__ bins,
              long long rows_stride, long long row_offset) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < nrow * nb; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(e / nrow);
    const long long r = e - static_cast<long long>(b) * nrow;
    for (int k = start[b]; k < start[b + 1]; ++k) {
      const BundleMember bm = mem[k];
      const double v = row_major ? static_cast<double>(X[r * ld + bm.real_index]) : static_cast<double>(X[static_cast<long long>(bm.real_index) * ld + r]);
      if (!d_off_mfb(v, bm)) continue;
      const FeatMeta m = meta[bm.inner];
      const unsigned bin = d_num_bin(v, m, ub + static_cast<size_t>(bm.inner) * 256, 1);
      if (bin == static_cast<unsigned>(m.default_bin)) continue;      // never written as a slot (d_bundle_slot needs bin != mfb)
      const int c = bundle_col[b];
      bins[(static_cast<size_t>(c >> 5) * rows_stride + row_offset + r) * 32 + (c & 31)] = static_cast<uint8_t>(d_bundle_slot(bin, bm.base, m.default_bin));
      break;
    }
  }
}

// ---------------------------------------------------------------- K1 gradients
// [UPSTREAM RegressionL2loss::GetGradients]
__global__ void k_grad_l2(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight,
                          float* __restrict__ g, float* __restrict__ h, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (weight) { g[i] = static_cast<float>((score[i] - label[i]) * weight[i]); h[i] = weight[i]; }
    else { g[i] = static_cast<float>(score[i] - label[i]); h[i] = 1.0f; }
  }
}
// [UPSTREAM RegressionHuberLoss / FairLoss / PoissonLoss / GammaLoss / TweedieLoss ::GetGradients]; kind 1..5
__global__ void k_grad_regvar(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight,
                              float* __restrict__ g, float* __restrict__ h, int n, int kind, double alpha, double c, double mds, double rho) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double s = score[i], lab = label[i];
    double gg, hh;
    if (kind == 1) { const double diff = s - lab; gg = fabs(diff) <= alpha ? diff : d_sign(diff) * alpha; hh = 1.0; }
    else if (kind == 2) { const double x = s - lab; gg = c * x / (fabs(x) + c); hh = c * c / ((fabs(x) + c) * (fabs(x) + c)); }
    else if (kind == 3) { gg = exp(s) - lab; hh = exp(s + mds); }
    else if (kind == 4) { gg = 1.0 - lab * exp(-s); hh = lab * exp(-s); }
    else { gg = -lab * exp((1 - rho) * s) + exp((2 - rho) * s); hh = -lab * (1 - rho) * exp((1 - rho) * s) + (2 - rho) * exp((2 - rho) * s); }
    if (weight) { gg *= weight[i]; hh *= weight[i]; }
    g[i] = static_cast<float>(gg); h[i] = static_cast<float>(hh);
  }
}
// [LightGBM RegressionL1loss / RegressionQuantileloss / RegressionMAPELOSS ::GetGradients]; kind 1 l1, 2 quantile, 3 mape
__global__ void k_grad_percentile(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight,
                                  const float* __restrict__ label_weight, float* __restrict__ g, float* __restrict__ h, int n, int kind, float alpha) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (kind == 2) {
      const float delta = static_cast<float>(score[i] - label[i]);
      const float gg = delta >= 0 ? (1.0f - alpha) : -alpha;
      g[i] = weight ? __fmul_rn(gg, weight[i]) : gg;
    } else {
      const double diff = score[i] - label[i];
      const int sgn = (diff > 0.0) - (diff < 0.0);
      if (kind == 1) g[i] = weight ? static_cast<float>(sgn * static_cast<double>(weight[i])) : static_cast<float>(sgn);
      else g[i] = static_cast<float>(sgn * static_cast<double>(label_weight[i]));
    }
    h[i] = weight ? weight[i] : 1.0f;
  }
}
// [UPSTREAM BinaryLogloss::GetGradients]
__global__ void k_grad_binary(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight,
                              float* __restrict__ g, float* __restrict__ h, int n, double sigmoid, double w_neg, double w_pos) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int is_pos = label[i] > 0;
    const double lab = is_pos ? 1.0 : -1.0;
    const double lw = is_pos ? w_pos : w_neg;
    const double response = -lab * sigmoid / (1.0 + exp(lab * sigmoid * score[i]));
    const double abs_response = fabs(response);
    double gg = response * lw, hh = abs_response * (sigmoid - abs_response) * lw;
    if (weight) { gg *= weight[i]; hh *= weight[i]; }
    g[i] = static_cast<float>(gg); h[i] = static_cast<float>(hh);
  }
}
// [UPSTREAM MulticlassOVA::GetGradients]: class k is a BinaryLogloss on (label == k); cw = per-class {w_neg, w_pos}, need = per-class need_train
__global__ void k_grad_ova(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight, float* __restrict__ g,
                           float* __restrict__ h, int n, int K, double sigmoid, const double* __restrict__ cw, const uint8_t* __restrict__ need) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int li = static_cast<int>(label[i]);
    for (int k = 0; k < K; ++k) {
      if (!need[k]) continue;
      const size_t id = static_cast<size_t>(n) * k + i;
      const int is_pos = li == k;
      const double lab = is_pos ? 1.0 : -1.0;
      const double lw = cw[2 * k + is_pos];
      const double response = -lab * sigmoid / (1.0 + exp(lab * sigmoid * score[id]));
      const double abs_response = fabs(response);
      double gg = response * lw, hh = abs_response * (sigmoid - abs_response) * lw;
      if (weight) { gg *= weight[i]; hh *= weight[i]; }
      g[id] = static_cast<float>(gg); h[id] = static_cast<float>(hh);
    }
  }
}
// [UPSTREAM CrossEntropy::GetGradients]: labels are probabilities
__global__ void k_grad_xent(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight, float* __restrict__ g,
                            float* __restrict__ h, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double z = 1.0 / (1.0 + exp(-score[i]));
    double gg = z - label[i], hh = z * (1.0 - z);
    if (weight) { gg *= weight[i]; hh *= weight[i]; }
    g[i] = static_cast<float>(gg); h[i] = static_cast<float>(hh);
  }
}
// [UPSTREAM MulticlassSoftmax::GetGradients]; score/g/h are class-major [K][n]
__global__ void k_grad_softmax(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight,
                               float* __restrict__ g, float* __restrict__ h, int n, int K, double factor) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double wmax = score[i];
    for (int k = 1; k < K; ++k) wmax = fmax(wmax, score[static_cast<size_t>(n) * k + i]);
    double wsum = 0;
    for (int k = 0; k < K; ++k) wsum += exp(score[static_cast<size_t>(n) * k + i] - wmax);
    const int lab = static_cast<int>(label[i]);
    const double w = weight ? weight[i] : 1.0;
    for (int k = 0; k < K; ++k) {
      double p = exp(score[static_cast<size_t>(n) * k + i] - wmax) / wsum;
      double gg = (lab == k) ? p - 1.0 : p, hh = factor * p * (1.0 - p);
      if (weight) { gg *= w; hh *= w; }
      g[static_cast<size_t>(n) * k + i] = static_cast<float>(gg);
      h[static_cast<size_t>(n) * k + i] = static_cast<float>(hh);
    }
  }
}

// The score a ranking objective sees for row i.  [UPSTREAM 4.1, from knowledge] unbiased lambdarank: with a position field, both ranking
// objectives take their gradients at s_i + b[id_i], the row's position factor added; pos_id null is the plain score.
__device__ __forceinline__ double d_rank_score(const double* __restrict__ score, const int* __restrict__ pos_id, const double* __restrict__ pos_bias,
                                               int i) {
  double s = score[i];
  if (pos_id) s += pos_bias[pos_id[i]];
  return s;
}

// [UPSTREAM LambdarankNDCG::GetGradientsForOneQuery] — one block per query (K2).
// Sorting: stable rank by score descending (rank counting out of shared memory; queries are ~100 docs).
// Pairs (i, j), i < min(truncation, cnt-1), j > i, are evaluated ONCE, tile by tile over j, by all threads (balanced) into a
// shared-memory matrix M[i][j] = (+-p_lambda, p_hessian) as fp32; then one thread per DOCUMENT adds its entries in the reference's own
// pair order — for document p: (0,p), (1,p) .. (p-1,p), then (p,p+1) .. (p,cnt-1) — with fp32 adds on a score_t accumulator.  No atomics
// (shared-memory float atomicAdd is a CAS loop on sm_90a), no double evaluation (the pair math is fp64 with a software division and a
// table look-up: the first version of this kernel, which evaluated every pair once per side, was FP64-bound at 2.4 ms per 50k queries),
// and every document's lambda / hessian is the same sequence of fp32 additions as the sequential reference: gradients are reproducible
// and equal to the oracle's up to the fp64 rounding of the normalisation factor.  discount[] = 1 / log2(2 + pos) is the host-computed
// table the reference uses (DCGCalculator), not a device log2.
constexpr int kLrThreads = 128;
__host__ __device__ inline int lr_tile(int truncation) {          // j-tile width: M = truncation x (tile + 1) float2 within 48 KB
  int t = (48 * 1024 / 8) / max(truncation, 1) - 1;
  t = min(t, 128);                 // queries are ~100 documents: one tile, and 20 KB per block keeps 8+ blocks per SM
  return max(t & ~31, 32);
}
__global__ void __launch_bounds__(kLrThreads)
k_grad_lambdarank(const double* __restrict__ score, const int* __restrict__ pos_id, const double* __restrict__ pos_bias,
                  const float* __restrict__ label, const float* __restrict__ weight,
                  const int* __restrict__ qb, int nq, const double* __restrict__ inv_max_dcg, const double* __restrict__ label_gain,
                  const double* __restrict__ discount, const float* __restrict__ sig_table, int sig_bins, double min_in, double max_in,
                  double idx_factor, double sigmoid, int truncation, int norm, float* __restrict__ g, float* __restrict__ h, int max_q) {
  extern __shared__ unsigned char lr_smem[];
  double* r_score = reinterpret_cast<double*>(lr_smem);                  // [max_q] scores in document order
  double* s_score = r_score + max_q;                                     // [max_q] scores by sorted position
  int* s_lab = reinterpret_cast<int*>(s_score + max_q);                  // label by sorted position
  int* s_orig = s_lab + max_q;                                           // document index by sorted position
  float* s_lam = reinterpret_cast<float*>(s_orig + max_q);               // accumulators by sorted position
  float* s_hes = s_lam + max_q;
  float2* M = reinterpret_cast<float2*>(s_hes + max_q);                  // [truncation][T + 1]; 32 * max_q bytes precede it: 8-byte aligned
  __shared__ double s_part[kLrThreads];
  const int T = lr_tile(truncation), TS = T + 1;
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const int start = qb[q], cnt = qb[q + 1] - start;
    __syncthreads();
    // two loops rather than d_rank_score's test per row: one loop holds 8 more registers through the whole kernel
    if (pos_id) for (int i = threadIdx.x; i < cnt; i += blockDim.x) r_score[i] = score[start + i] + pos_bias[pos_id[start + i]];
    else for (int i = threadIdx.x; i < cnt; i += blockDim.x) r_score[i] = score[start + i];
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const double si = r_score[i];
      int rank = 0;
      for (int j = 0; j < cnt; ++j) {
        const double sj = r_score[j];
        rank += (sj > si) || (sj == si && j < i);
      }
      s_score[rank] = si; s_lab[rank] = static_cast<int>(label[start + i]); s_orig[rank] = i;
      s_lam[rank] = 0.f; s_hes[rank] = 0.f;
    }
    __syncthreads();
    const double imd = inv_max_dcg[q];
    const double best_score = s_score[0];
    int worst_idx = cnt - 1;
    if (worst_idx > 0 && s_score[worst_idx] == kNegInf) worst_idx -= 1;
    const double worst_score = s_score[worst_idx];
    const bool do_div = norm && best_score != worst_score;
    const int teff = min(truncation, cnt - 1);          // pairs exist for i < teff
    double local_sum = 0.0;
    for (int j0 = 0; j0 < cnt; j0 += T) {
      const int tcnt = min(T, cnt - j0);
      // ---- phase A: every pair of the tile once
      for (int e = threadIdx.x; e < teff * tcnt; e += blockDim.x) {
        const int i = e / tcnt, jj = e - i * tcnt, j = j0 + jj;
        float2 m = make_float2(0.f, 0.f);
        if (j > i) {
          const double sci = s_score[i], scj = s_score[j];
          const int li = s_lab[i], lj = s_lab[j];
          if (sci != kNegInf && scj != kNegInf && li != lj) {
            const bool ih = li > lj;                     // position i holds the higher label
            const int hr = ih ? i : j, lr = ih ? j : i;
            const double delta_score = ih ? sci - scj : scj - sci;
            const double dcg_gap = label_gain[ih ? li : lj] - label_gain[ih ? lj : li];
            const double paired_discount = fabs(discount[hr] - discount[lr]);
            double delta = dcg_gap * paired_discount * imd;
            if (do_div) delta /= (0.01f + fabs(delta_score));
            double pl;
            if (delta_score <= min_in) pl = sig_table[0];
            else if (delta_score >= max_in) pl = sig_table[sig_bins - 1];
            else pl = sig_table[static_cast<size_t>((delta_score - min_in) * idx_factor)];
            double ph = pl * (1.0f - pl);
            pl *= -sigmoid * delta;
            ph *= sigmoid * sigmoid * delta;
            local_sum -= 2 * pl;
            const float fl = static_cast<float>(pl);
            m = make_float2(ih ? fl : -fl, static_cast<float>(ph));      // lambdas[i] += m.x, lambdas[j] -= m.x (x - y == x + (-y) exactly)
          }
        }
        M[i * TS + jj] = m;
      }
      __syncthreads();
      // ---- phase B: one thread per document, the reference's order of additions
      for (int p = threadIdx.x; p < cnt; p += blockDim.x) {
        const bool as_j = p >= j0 && p < j0 + tcnt, as_i = p < teff && p + 1 < j0 + tcnt;
        if (!as_j && !as_i) continue;
        float lam = s_lam[p], hes = s_hes[p];
        if (as_j) {
          const int ilim = min(p, teff);
          for (int i = 0; i < ilim; ++i) { const float2 m = M[i * TS + (p - j0)]; lam = __fsub_rn(lam, m.x); hes = __fadd_rn(hes, m.y); }
        }
        if (as_i) {
          for (int j = max(j0, p + 1); j < j0 + tcnt; ++j) { const float2 m = M[p * TS + (j - j0)]; lam = __fadd_rn(lam, m.x); hes = __fadd_rn(hes, m.y); }
        }
        s_lam[p] = lam; s_hes[p] = hes;
      }
      __syncthreads();
    }
    s_part[threadIdx.x] = local_sum;
    __syncthreads();
    double sum_lambdas = 0.0;
    if (norm) for (int t = 0; t < static_cast<int>(blockDim.x); ++t) sum_lambdas += s_part[t];      // fixed order: reproducible
    double nf = 1.0;
    const bool do_norm = norm && sum_lambdas > 0;
    if (do_norm) nf = log2(1 + sum_lambdas) / sum_lambdas;
    for (int r = threadIdx.x; r < cnt; r += blockDim.x) {
      float lam = s_lam[r], hes = s_hes[r];
      if (do_norm) { lam = static_cast<float>(lam * nf); hes = static_cast<float>(hes * nf); }
      const int o = start + s_orig[r];
      if (weight) { lam = static_cast<float>(lam * weight[o]); hes = static_cast<float>(hes * weight[o]); }
      g[o] = lam; h[o] = hes;
    }
  }
}

// [UPSTREAM RankXENDCG::GetGradientsForOneQuery] — one block per query, like k_grad_lambdarank.  Every query owns an LCG
// (x <- 214013 x + 2531011, float = ((x >> 16) & 0x7fff) / 32768) seeded objective_seed + q; document i takes its (i+1)-th output, which
// the jump table gives directly (x_{i+1} = jump_mul[i] * x0 + jump_add[i], as k_bag_draw).  rho (softmax of the scores) and the params
// of the three Taylor terms live in `scratch` [2][n] fp64 at the query's rows.  The four sums (softmax denominator, sum of params,
// sum_l1, sum_l2) are taken by one thread in document order, the reference's order, so the kernel differs from it only where the
// device exp differs from the host's.  Products that are added are rounded separately (__dmul_rn): the reference does not fuse them.
// advance != 0 (a training iteration) moves every query's state on by cnt draws; GetGradients reads without advancing.
__device__ __forceinline__ float d_lcg_float(unsigned x) { return static_cast<float>((x >> 16) & 0x7FFFu) / 32768.0f; }
constexpr int kXeThreads = 128;
__global__ void __launch_bounds__(kXeThreads)
k_grad_xendcg(const double* __restrict__ score, const int* __restrict__ pos_id, const double* __restrict__ pos_bias, const float* __restrict__ label,
              const float* __restrict__ weight, const int* __restrict__ qb,
              int nq, unsigned* __restrict__ lcg_state, const unsigned* __restrict__ jump_mul, const unsigned* __restrict__ jump_add, int advance,
              double* __restrict__ scratch, size_t n, float* __restrict__ g, float* __restrict__ h) {
  __shared__ double s_sum;
  double* rho = scratch;
  double* params = scratch + n;
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const int start = qb[q], cnt = qb[q + 1] - start;
    if (cnt <= 1) {              // no draws
      if (cnt == 1 && threadIdx.x == 0) { g[start] = 0.0f; h[start] = 0.0f; }
      continue;
    }
    const unsigned x0 = lcg_state[q];
    double* r = rho + start;
    double* pa = params + start;
    // softmax: max (order-free), exp, denominator in document order
    double wmax = -INFINITY;
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) wmax = fmax(wmax, d_rank_score(score, pos_id, pos_bias, start + i));
    for (int o = 16; o; o >>= 1) wmax = fmax(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    __shared__ double s_max[kXeThreads / 32];
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = wmax;
    __syncthreads();
    wmax = s_max[0];
    for (int w = 1; w < kXeThreads / 32; ++w) wmax = fmax(wmax, s_max[w]);
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      r[i] = exp(d_rank_score(score, pos_id, pos_bias, start + i) - wmax);
      const unsigned x = jump_mul[i] * x0 + jump_add[i];
      pa[i] = ldexp(1.0, static_cast<int>(label[start + i])) - static_cast<double>(d_lcg_float(x));
    }
    __syncthreads();
    if (threadIdx.x == 0) { double s = 0.0; for (int i = 0; i < cnt; ++i) s += r[i]; s_sum = s; }
    __syncthreads();
    const double wsum = s_sum;
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) r[i] /= wsum;
    if (threadIdx.x == 0) { double s = 0.0; for (int i = 0; i < cnt; ++i) s += pa[i]; s_sum = s; }
    __syncthreads();
    const double inv = 1.0 / fmax(kEps, s_sum);
    __syncthreads();
    // first-order term
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const double t = __dadd_rn(-__dmul_rn(pa[i], inv), r[i]);
      g[start + i] = static_cast<float>(t);
      pa[i] = t / (1.0 - r[i]);
    }
    __syncthreads();
    if (threadIdx.x == 0) { double s = 0.0; for (int i = 0; i < cnt; ++i) s += pa[i]; s_sum = s; }
    __syncthreads();
    const double sum_l1 = s_sum;
    __syncthreads();
    // second-order term
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const double t = r[i] * (sum_l1 - pa[i]);
      g[start + i] = __fadd_rn(g[start + i], static_cast<float>(t));
      pa[i] = t / (1.0 - r[i]);
    }
    __syncthreads();
    if (threadIdx.x == 0) { double s = 0.0; for (int i = 0; i < cnt; ++i) s += pa[i]; s_sum = s; }
    __syncthreads();
    const double sum_l2 = s_sum;
    // third-order term, hessian, row weight (score_t * label_t)
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      float lam = __fadd_rn(g[start + i], static_cast<float>(r[i] * (sum_l2 - pa[i])));
      float hes = static_cast<float>(r[i] * (1.0 - r[i]));
      if (weight) { lam = __fmul_rn(lam, weight[start + i]); hes = __fmul_rn(hes, weight[start + i]); }
      g[start + i] = lam; h[start + i] = hes;
    }
    if (advance && threadIdx.x == 0) lcg_state[q] = jump_mul[cnt - 1] * x0 + jump_add[cnt - 1];
    __syncthreads();
  }
}

// [UPSTREAM CrossEntropyLambda::GetGradients]: labels are probabilities; with weights, the weight enters the link 1 - exp(-w log1p(e^s))
__global__ void k_grad_xentlambda(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight,
                                  float* __restrict__ g, float* __restrict__ h, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double y = label[i];
    if (!weight) {
      const double z = 1.0 / (1.0 + exp(-score[i]));
      g[i] = static_cast<float>(z - y); h[i] = static_cast<float>(z * (1.0 - z));
      continue;
    }
    const double w = weight[i], epf = exp(score[i]), hhat = log1p(epf), z = 1.0 - exp(-w * hhat), enf = 1.0 / epf;
    g[i] = static_cast<float>((1.0 - y / z) * w / (1.0 + enf));
    const double c = 1.0 / (1.0 - z);
    double d = 1.0 + epf;
    const double a = w * epf / (d * d);
    d = c - 1.0;
    const double b = (c / (d * d)) * (__dadd_rn(1.0, __dmul_rn(w, epf)) - c);
    h[i] = static_cast<float>(a * __dadd_rn(1.0, __dmul_rn(y, b)));
  }
}

// ---------------------------------------------------------------- quantisation + root sums (K3)
// one value's word on K3's fixed-point grid: q = rint(x * 2^e), e from k_set_scale (the quantisation, the renewed and the refit leaf sums)
__device__ __forceinline__ long long d_fixed(float x, int e) { return __double2ll_rn(ldexp(static_cast<double>(x), e)); }
__global__ void k_absmax(const float* __restrict__ g, const float* __restrict__ h, int n, TreeCtrl* ctrl) {
  float mg = 0.f, mh = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    mg = fmaxf(mg, fabsf(g[i])); mh = fmaxf(mh, fabsf(h[i]));
  }
  for (int o = 16; o; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&ctrl->absmax_bits[0], __float_as_uint(mg));
    atomicMax(&ctrl->absmax_bits[1], __float_as_uint(mh));
  }
}
// exponents so that |q| < 2^35:  e = 34 - ilogb(max)
__global__ void k_set_scale(TreeCtrl* ctrl, int const_hessian, double hess_const) {
  float mg = __uint_as_float(ctrl->absmax_bits[0]), mh = __uint_as_float(ctrl->absmax_bits[1]);
  int eg = (mg > 0.f && isfinite(mg)) ? 34 - ilogbf(mg) : 0;
  int eh = (mh > 0.f && isfinite(mh)) ? 34 - ilogbf(mh) : 0;
  eg = max(min(eg, 1000), -1000); eh = max(min(eh, 1000), -1000);
  ctrl->exp_g = eg; ctrl->exp_h = eh;
  ctrl->inv_g = ldexp(1.0, -eg);
  ctrl->inv_h = const_hessian ? hess_const : ldexp(1.0, -eh);
  ctrl->root_q[0] = 0; ctrl->root_q[1] = 0; ctrl->root_q[2] = 0; ctrl->root_q[3] = 0;
}

// Position row ids (Objective): ids[i] = the index of pos[i] in the sorted distinct values `values` [P], which hold every value of pos
__global__ void __launch_bounds__(256)
k_position_ids(const int* __restrict__ pos, int n, const int* __restrict__ values, int P, int* __restrict__ ids) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int v = pos[i];
    int lo = 0, hi = P - 1;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (values[mid] < v) lo = mid + 1; else hi = mid; }
    ids[i] = lo;
  }
}
// [UPSTREAM 4.1 RankingObjective::UpdatePositionBiasFactors, from knowledge] one thread per position id p, at k_refit_leaf_sums' (all-reduced)
// sums of the weighted g and h over the rows of p (sums [3][P]: Q_g, Q_h, rows):
//   d1 = -sum_g - b_p * reg * cnt,  d2 = -sum_h - reg * cnt,  b_p += learning_rate * d1 / (|d2| + 0.001)
// sum_g = Q_g 2^-e_g and sum_h = Q_h 2^-e_h on K3's grid.  Every fp64 operation is rounded on its own, in this order, so a restatement
// can follow it bit for bit.
__global__ void k_position_bias_update(const long long* __restrict__ sums, int P, const TreeCtrl* __restrict__ ctrl, double learning_rate,
                                       double reg, double* __restrict__ bias) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const double sg = __dmul_rn(static_cast<double>(sums[p]), ldexp(1.0, -ctrl->exp_g));
  const double sh = __dmul_rn(static_cast<double>(sums[P + p]), ldexp(1.0, -ctrl->exp_h));
  const double cnt = static_cast<double>(sums[2 * P + p]);
  const double b = bias[p];
  const double d1 = __dsub_rn(-sg, __dmul_rn(__dmul_rn(b, reg), cnt));
  const double d2 = __dsub_rn(-sh, __dmul_rn(reg, cnt));
  bias[p] = __dadd_rn(b, __ddiv_rn(__dmul_rn(learning_rate, d1), __dadd_rn(fabs(d2), 0.001)));
}
// a 256-thread block's share of the root sums: sum q_g, sum q_h over its in-bag rows, and (block 0) the rows of the root
__device__ __forceinline__ void d_add_root_sums(long long sg, long long sh, TreeCtrl* ctrl, const uint8_t* in_bag, int bag_count, int n) {
  for (int o = 16; o; o >>= 1) { sg += __shfl_xor_sync(0xffffffffu, sg, o); sh += __shfl_xor_sync(0xffffffffu, sh, o); }
  __shared__ long long s_g[8], s_h[8];
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_g[warp] = sg; s_h[warp] = sh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long a = 0, b = 0;
    for (int w = 0; w < 8; ++w) { a += s_g[w]; b += s_h[w]; }
    atomicAdd(reinterpret_cast<unsigned long long*>(&ctrl->root_q[0]), static_cast<unsigned long long>(a));
    atomicAdd(reinterpret_cast<unsigned long long*>(&ctrl->root_q[1]), static_cast<unsigned long long>(b));
    if (blockIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&ctrl->root_q[2]), static_cast<unsigned long long>(in_bag ? bag_count : n));
  }
}
__global__ void __launch_bounds__(256)
k_quantize(const float* __restrict__ g, const float* __restrict__ h, int n, int4* __restrict__ qgh, TreeCtrl* ctrl, int const_hessian,
           const uint8_t* __restrict__ in_bag, int bag_count) {
  const int eg = ctrl->exp_g, eh = ctrl->exp_h;
  long long sg = 0, sh = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    long long qg = d_fixed(g[i], eg);
    int4 q;
    q.x = static_cast<int>(qg >> kLoBits); q.y = static_cast<int>(qg & ((1LL << kLoBits) - 1));
    long long qh;
    if (const_hessian) { qh = 1; q.z = 1; q.w = 0; }
    else { qh = d_fixed(h[i], eh); q.z = static_cast<int>(qh >> kLoBits); q.w = static_cast<int>(qh & ((1LL << kLoBits) - 1)); }
    qgh[i] = q;
    if (!in_bag || in_bag[i]) { sg += qg; sh += qh; }       // root sums run over the in-bag rows only
  }
  d_add_root_sums(sg, sh, ctrl, in_bag, bag_count, n);
}

// ---------------------------------------------------------------- quantised training (use_quantized_grad), K3's discretisation
// [UPSTREAM 4.x GradientDiscretizer::DiscretizeGradients], restated from knowledge: per tree, g and h become a few integer levels,
// q_g in [-floor(B/2), floor(B/2)] at scale s_g = max|g| / floor(B/2) and q_h in [-B, B] at s_h = max|h| / B (B = num_grad_quant_bins;
// a zero maximum gives scale 1).  Constant hessians keep q_h = 1 (the count plane).  tests/quant_ref.py restates every fp64 operation.
// The draws of stochastic rounding: u in [0, 1) from a counter-based hash of (data_random_seed, tree index, rank-local row, g or h), so
// nothing carries from tree to tree and any tree's draws follow from its key whatever the launch shape.  (LightGBM's own stream is not
// reproduced.)
__device__ __forceinline__ unsigned long long d_mix64(unsigned long long z) {      // splitmix64's finaliser
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ double d_quant_uniform(int seed, int tree, int row, int which) {
  unsigned long long z = d_mix64(static_cast<unsigned long long>(static_cast<unsigned>(seed)));
  z = d_mix64(z ^ static_cast<unsigned long long>(static_cast<unsigned>(tree)));
  z = d_mix64(z ^ (2ull * static_cast<unsigned>(row) + static_cast<unsigned>(which)));
  return static_cast<double>(z >> 11) * 0x1.0p-53;
}
// One value's level: v = x / s; with stochastic rounding trunc(v + sign(v) u), else v rounded half away from zero; clamped to [-lim, lim]
__device__ __forceinline__ int d_discretize(float x, double s, int lim, int stochastic, double u) {
  const double v = static_cast<double>(x) / s;
  double q;
  if (stochastic) {
    q = trunc(v + d_sign(v) * u);
  } else {
    q = trunc(v);
    if (fabs(v - q) >= 0.5) q += d_sign(v);
  }
  return static_cast<int>(fmin(fmax(q, static_cast<double>(-lim)), static_cast<double>(lim)));
}
// after k_set_scale (whose exponents the leaf renewal keeps using): the scales of the discretised words
__global__ void k_set_quant_scale(TreeCtrl* ctrl, int const_hessian, int quant_bins) {
  const float mg = __uint_as_float(ctrl->absmax_bits[0]), mh = __uint_as_float(ctrl->absmax_bits[1]);
  ctrl->inv_g = (mg > 0.f && isfinite(mg)) ? static_cast<double>(mg) / (quant_bins / 2) : 1.0;
  if (!const_hessian) ctrl->inv_h = (mh > 0.f && isfinite(mh)) ? static_cast<double>(mh) / quant_bins : 1.0;
}
// q into K3's fixed-point words (the same {g_hi, g_lo, h_hi, h_lo} layout, so every later kernel reads them as it reads k_quantize's) and
// the root sums over the in-bag rows.  tree: iteration * trees per iteration + class.
__global__ void __launch_bounds__(256)
k_quantize_discrete(const float* __restrict__ g, const float* __restrict__ h, int n, int4* __restrict__ qgh, TreeCtrl* ctrl, int const_hessian,
                    const uint8_t* __restrict__ in_bag, int bag_count, int quant_bins, int stochastic, int seed, int tree) {
  const double sg_scale = ctrl->inv_g, sh_scale = ctrl->inv_h;
  long long sg = 0, sh = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int qg = d_discretize(g[i], sg_scale, quant_bins / 2, stochastic, stochastic ? d_quant_uniform(seed, tree, i, 0) : 0.0);
    const int qh = const_hessian ? 1 : d_discretize(h[i], sh_scale, quant_bins, stochastic, stochastic ? d_quant_uniform(seed, tree, i, 1) : 0.0);
    int4 q;
    q.x = qg >> kLoBits; q.y = qg & ((1 << kLoBits) - 1);
    if (const_hessian) { q.z = 1; q.w = 0; }
    else { q.z = qh >> kLoBits; q.w = qh & ((1 << kLoBits) - 1); }
    qgh[i] = q;
    if (!in_bag || in_bag[i]) { sg += qg; sh += qh; }
  }
  d_add_root_sums(sg, sh, ctrl, in_bag, bag_count, n);
}

// quant_train_renew_leaf ([UPSTREAM 4.x GradientDiscretizer::RenewIntGradTreeOutput], from knowledge): each leaf's true in-bag sums of
// g and h on K3's 36-bit fixed-point grid (k_set_scale's exponents), so they are exact and order-independent and ranks agree bit for bit.
// grid x = num_leaves * blocks_per_leaf: block b sums part b % blocks_per_leaf of leaf b / blocks_per_leaf.  sums: [num_leaves][2], zeroed.
__global__ void __launch_bounds__(256)
k_quant_leaf_sums(const TreeCtrl* __restrict__ ctrl, const LeafState* __restrict__ leaves, const int* __restrict__ idx0,
                  const int* __restrict__ idx1, const float* __restrict__ g, const float* __restrict__ h, int const_hessian,
                  int blocks_per_leaf, long long* __restrict__ sums) {
  const int l = blockIdx.x / blocks_per_leaf, part = blockIdx.x - l * blocks_per_leaf;
  if (l >= ctrl->num_leaves) return;
  const LeafState& L = leaves[l];
  const int* src = L.buf ? idx1 : idx0;
  const int eg = ctrl->exp_g, eh = ctrl->exp_h;
  long long sg = 0, sh = 0;
  for (int i = part * blockDim.x + threadIdx.x; i < L.count; i += blocks_per_leaf * blockDim.x) {
    const int r = L.identity ? (L.begin + i) : src[L.begin + i];
    sg += d_fixed(g[r], eg);
    sh += const_hessian ? 1 : d_fixed(h[r], eh);
  }
  for (int o = 16; o; o >>= 1) { sg += __shfl_xor_sync(0xffffffffu, sg, o); sh += __shfl_xor_sync(0xffffffffu, sh, o); }
  if ((threadIdx.x & 31) == 0 && (sg | sh)) {
    atomicAdd(reinterpret_cast<unsigned long long*>(&sums[2 * l]), static_cast<unsigned long long>(sg));
    atomicAdd(reinterpret_cast<unsigned long long*>(&sums[2 * l + 1]), static_cast<unsigned long long>(sh));
  }
}
// leaf_value = d_calc_output at the (all-reduced) true sums; leaf_weight, internal values and counts keep the quantised sums.  A leaf
// whose true h sum + lambda_l2 is 0 (custom hessians can cancel; the scans chose the split on the quantised sums) keeps its quantised
// output instead of an inf or NaN.
__global__ void k_quant_renew_apply(const TreeCtrl* __restrict__ ctrl, TreeDev tree, const long long* __restrict__ sums, int const_hessian,
                                    SplitParams p) {
  const int nl = ctrl->num_leaves;
  const double ig = ldexp(1.0, -ctrl->exp_g), ih = const_hessian ? 1.0 : ldexp(1.0, -ctrl->exp_h);
  for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < nl; l += gridDim.x * blockDim.x) {
    const double sh = static_cast<double>(sums[2 * l + 1]) * ih;
    if (sh + p.l2 != 0.0) tree.leaf_value[l] = d_calc_output(static_cast<double>(sums[2 * l]) * ig, sh, p);
  }
}

// ---------------------------------------------------------------- tree init / round controller
__global__ void __launch_bounds__(256)
k_tree_init(TreeCtrl* ctrl, LeafState* leaves, TreeDev tree, uint8_t* flags, SplitParams p, int n_local, const uint8_t* feature_used,
            int root_is_bag, unsigned col_state) {
  for (int u = threadIdx.x; u < p.nf_pad; u += blockDim.x) flags[u] = (u < p.nf && (!feature_used || feature_used[u])) ? 1 : 0;
  for (int l = threadIdx.x; l < p.num_leaves; l += blockDim.x) {
    leaves[l].best.gain = kNegInf; leaves[l].best.feature = -1;
    tree.leaf_parent[l] = -1; tree.leaf_depth[l] = 0; tree.leaf_value[l] = 0; tree.leaf_weight[l] = 0; tree.leaf_count[l] = 0;
  }
  if (threadIdx.x == 0) {
    LeafState& r = leaves[0];
    r.begin = 0; r.count = n_local; r.buf = 0; r.depth = 0; r.identity = root_is_bag ? 0 : 1; r.hist_slot = 0; r.parent_node = -1;
    r.mono_min = kNegInf; r.mono_max = -kNegInf; r.inter_mask = ~0ull;
    r.global_count = static_cast<int>(ctrl->root_q[2]);
    r.sum_g = static_cast<double>(ctrl->root_q[0]) * ctrl->inv_g;
    r.sum_h = static_cast<double>(ctrl->root_q[1]) * ctrl->inv_h;
    // path smoothing: the root's parent_output is its own output, from the all-reduced sums without the scans' 2 kEpsilon; smoothing
    // toward it gives it back
    r.output = d_calc_output(r.sum_g, r.sum_h, p);
    ctrl->num_leaves = 1; ctrl->left_leaf = 0; ctrl->right_leaf = -1; ctrl->smaller = 0; ctrl->larger = -1;
    ctrl->go = 0; ctrl->finished = 0; ctrl->split_leaf = -1; ctrl->pending = 0; ctrl->round = 0; ctrl->trace_rows = 0;
    ctrl->col_state = col_state; ctrl->forced_next = 0;
    *tree.num_leaves = 1;
  }
}

// The constraints of the two children when the round controller applies a split of leaf L into L and R.  Out of line to keep it off the
// partition kernel's registers.
// Monotone constraints ([UPSTREAM] BasicLeafConstraints::Update): both children inherit the parent's bounds; a numerical split on a
// monotone feature narrows them at mid = (left_out + right_out) / 2 — the left child's max and the right child's min for +1, the mirror
// for -1.
// Interaction constraints (interaction != 0): both children's set mask is the parent's & the split feature's sets_of word.
// Path smoothing: each child keeps its output as the parent_output of its own scans.
__device__ __noinline__ void d_constrain_children(LeafState& L, LeafState& R, int monotone_type, int is_cat, double left_out, double right_out,
                                                  int interaction, const unsigned long long& inter_sets) {
  L.output = left_out; R.output = right_out;
  R.mono_min = L.mono_min; R.mono_max = L.mono_max;
  if (monotone_type != 0 && !is_cat) {
    const double mid = (left_out + right_out) / 2.0;
    if (monotone_type > 0) { L.mono_max = fmin(L.mono_max, mid); R.mono_min = fmax(R.mono_min, mid); }
    else { L.mono_min = fmax(L.mono_min, mid); R.mono_max = fmin(R.mono_max, mid); }
  }
  if (interaction) { const unsigned long long m = L.inter_mask & inter_sets; L.inter_mask = m; R.inter_mask = m; }
}

// Applies the split chosen in the previous round (Tree::Split + leaf bookkeeping, using the TRUE row
// counts in the serial learner and the hessian-reconstructed global counts in the data-parallel one),
// then runs SerialTreeLearner::BeforeFindBestSplit for the coming round.  One block; thread 0 does the bookkeeping, all threads copy
// the inherited is_splittable flags.  Runs as its own kernel before a tree's first round and, for every later round, in the last
// block of the partition kernel of the previous round (k_partition) — one launch and one kernel boundary less per split.
__device__ __forceinline__ void
d_round_ctl(TreeCtrl* ctrl, LeafState* leaves, const TreeDev& tree, uint8_t* flags, const FeatMeta* __restrict__ meta, const SplitParams& p, int last,
            int* s_copy) {       // s_copy: 2 shared ints
  if (threadIdx.x == 0) {
    s_copy[0] = -1; s_copy[1] = -1;
    if (ctrl->pending) {
      ctrl->pending = 0;
      const int leaf = ctrl->split_leaf, nl = ctrl->new_leaf;
      LeafState& L = leaves[leaf];
      LeafState& R = leaves[nl];
      L.qpar[0] = R.qpar[0] = L.qtot[0]; L.qpar[1] = R.qpar[1] = L.qtot[1];
      LeafBest b = L.best;
      // written by another block of the same kernel when this runs as the tail of k_partition: read through L2
      const int true_left = __ldcg(&ctrl->part_left_total), true_right = ctrl->part_count - true_left;
      if (!p.parallel) { b.left_count = true_left; b.right_count = true_right; }
      // Tree::Split
      const int node = ctrl->num_leaves - 1;
      const int parent = tree.leaf_parent[leaf];
      if (parent >= 0) {
        if (tree.left_child[parent] == ~leaf) tree.left_child[parent] = node; else tree.right_child[parent] = node;
      }
      tree.split_feature_inner[node] = b.feature;
      tree.split_gain[node] = static_cast<float>(b.gain + p.min_gain_to_split);
      tree.left_child[node] = ~leaf; tree.right_child[node] = ~nl;
      tree.leaf_parent[leaf] = node; tree.leaf_parent[nl] = node;
      tree.internal_weight[node] = tree.leaf_weight[leaf];
      tree.internal_value[node] = tree.leaf_value[leaf];
      tree.internal_count[node] = b.left_count + b.right_count;
      tree.leaf_value[leaf] = isnan(b.left_out) ? 0.0 : b.left_out;
      tree.leaf_weight[leaf] = b.left_h; tree.leaf_count[leaf] = b.left_count;
      tree.leaf_value[nl] = isnan(b.right_out) ? 0.0 : b.right_out;
      tree.leaf_weight[nl] = b.right_h; tree.leaf_count[nl] = b.right_count;
      tree.leaf_depth[nl] = tree.leaf_depth[leaf] + 1; tree.leaf_depth[leaf] += 1;
      const FeatMeta fm = meta[b.feature];
      if (b.is_cat) {
        tree.decision_type[node] = 1 | (fm.missing_type << 2);
        tree.threshold_bin[node] = 0;
      } else {
        tree.decision_type[node] = (b.default_left ? 2 : 0) | (fm.missing_type << 2);
        tree.threshold_bin[node] = b.threshold;
      }
      for (int wd = 0; wd < 8; ++wd) tree.cat_bits[node * 8 + wd] = b.is_cat ? b.cat_bits[wd] : 0u;
      tree.cat_list_len[node] = b.is_cat ? b.cat_list_len : 0;
      if (b.is_cat) for (int k = 0; k < b.cat_list_len && k < kCatListMax; ++k) tree.cat_list[node * kCatListMax + k] = b.cat_list[k];
      ctrl->num_leaves += 1; *tree.num_leaves = ctrl->num_leaves;
      // data partition bookkeeping: children live in the other index buffer
      const int dst_buf = L.identity ? 0 : (L.buf ^ 1);
      R.begin = L.begin + true_left; R.count = true_right; R.buf = dst_buf; R.identity = 0; R.depth = L.depth + 1;
      L.count = true_left; L.buf = dst_buf; L.identity = 0; L.depth += 1;
      L.global_count = b.left_count; R.global_count = b.right_count;
      L.sum_g = b.left_g; L.sum_h = b.left_h; R.sum_g = b.right_g; R.sum_h = b.right_h;
      d_constrain_children(L, R, b.monotone_type, b.is_cat, b.left_out, b.right_out, p.interaction, L.best.inter_sets);
      R.hist_slot = nl;
      L.best.gain = kNegInf; L.best.feature = -1; R.best.gain = kNegInf; R.best.feature = -1;
      ctrl->left_leaf = leaf; ctrl->right_leaf = nl;
    }
    ctrl->go = 0; ctrl->smaller = -1; ctrl->larger = -1; ctrl->split_leaf = -1;
    ctrl->hist_work.count = 0; ctrl->part_count = 0;
    if (!ctrl->finished && !last && ctrl->num_leaves < p.num_leaves) {
      const int ll = ctrl->left_leaf, rl = ctrl->right_leaf;
      bool go = true;
      if (p.max_depth > 0 && tree.leaf_depth[ll] >= p.max_depth) go = false;
      const int nl_cnt = leaves[ll].global_count, nr_cnt = rl >= 0 ? leaves[rl].global_count : 0;
      if (go && nr_cnt < p.min_data_in_leaf * 2 && nl_cnt < p.min_data_in_leaf * 2) go = false;
      if (!go) {
        leaves[ll].best.gain = kNegInf;
        if (rl >= 0) leaves[rl].best.gain = kNegInf;
      } else {
        int smaller = ll, larger = -1;
        if (rl >= 0) {
          if (nl_cnt < nr_cnt) { smaller = ll; larger = rl; } else { smaller = rl; larger = ll; }
          // parent's histogram sits in the slot of `ll`; the larger child inherits it
          if (larger == rl) { int t = leaves[ll].hist_slot; leaves[ll].hist_slot = leaves[rl].hist_slot; leaves[rl].hist_slot = t; }
          s_copy[0] = ll; s_copy[1] = rl;
        }
        ctrl->smaller = smaller; ctrl->larger = larger; ctrl->go = 1;
        const LeafState& S = leaves[smaller];
        ctrl->hist_work.begin = S.begin; ctrl->hist_work.count = S.count; ctrl->hist_work.use_idx = S.identity ? 0 : 1;
        ctrl->hist_work.buf = S.buf;       // K4 reads the row list from index buffer `buf`
        ctrl->smaller_rows = S.count;
        ctrl->trace_rows += S.count;
      }
    }
    ctrl->round += 1;
  }
  __syncthreads();
  if (s_copy[0] >= 0)   // children inherit the parent's per-feature is_splittable flags
    for (int u = threadIdx.x; u < p.nf_pad; u += blockDim.x) flags[static_cast<size_t>(s_copy[1]) * p.nf_pad + u] = flags[static_cast<size_t>(s_copy[0]) * p.nf_pad + u];
}
__global__ void __launch_bounds__(256)
k_round_ctl(TreeCtrl* ctrl, LeafState* leaves, TreeDev tree, uint8_t* flags, const FeatMeta* __restrict__ meta, SplitParams p,
            int last) {
  __shared__ int s_copy[2];
  d_round_ctl(ctrl, leaves, tree, flags, meta, p, last, s_copy);
}

// ---------------------------------------------------------------- K5/K6 split scan
// What k_scan (below) runs besides the numerical scan: the warp-level categorical search, and the pick step of its last block over the
// candidates of every feature, the wide ones from k_scan_wide included.  All sums are exact int64; gains are fp64.


// The larger leaf's block of a many-vs-many categorical feature: did the smaller leaf's scan of it draw?  Counts the smaller leaf's used
// bins (>= cat_smooth rebuilt rows, bin 0 excluded) in its histogram column `hist` (H), exactly as the smaller leaf's own scan counts
// them.  Called by every thread of the block; out of line to keep it off the scans' register budget.
__device__ __noinline__ bool d_smaller_drew_cat(const long long* __restrict__ hist, int num_bin, const LeafState& S, double inv_h,
                                                const SplitParams& p, int max_cat_threshold) {
  const double cnt_factor = S.global_count / (S.sum_h + 2 * kEpsD);
  int used_bin = 0;
  for (int b0 = 0; b0 < num_bin; b0 += blockDim.x) {      // the same trip count in every thread
    const int b = b0 + threadIdx.x;
    bool used = false;
    if (b >= 1 && b < num_bin) used = static_cast<int>(static_cast<double>(hist[b * 2 + 1]) * inv_h * cnt_factor + 0.5) >= p.cat_smooth;
    used_bin += __syncthreads_count(used);
  }
  return d_cat_rand_range(used_bin, max_cat_threshold) > 0;
}
// extra_trees, the larger leaf's block of feature m: did the smaller leaf's scan of it draw?  Both leaves hold the same pre-scan flag
// (inherited from their parent), so the smaller one scanned the feature too; it drew unless its range was empty, which only the
// many-vs-many categorical search decides from the data: the smaller leaf's used bins, counted in its histogram column `hist` (H).
// max_cat_threshold: the calling scan's.  Called by every thread of the block.
__device__ __forceinline__ bool d_smaller_drew(const long long* __restrict__ hist, const FeatMeta& m, const TreeCtrl* ctrl, const LeafState* leaves,
                                               const SplitParams& p, int max_cat_threshold) {
  if (!m.is_categorical) return m.num_bin > 2;
  if (m.num_bin <= p.max_cat_to_onehot) return m.num_bin > 1;
  return d_smaller_drew_cat(hist, m.num_bin, leaves[ctrl->smaller], ctrl->inv_h, p, max_cat_threshold);
}

// The many-vs-many walk of FindBestThresholdCategoricalInner [UPSTREAM] from one end of the ranked used bins: at most max_num_cat bins
// are added to the left side, with the sequential code's skip (continue) and stop (break) rules.  next(&g, &h) gives the next bin's sums
// in walk order; visit(i, slg, slh, srh, left_count) is called for every prefix (i + 1 bins) whose gain the reference evaluates.
template <bool kExtra, typename Next, typename Visit>
__device__ __forceinline__ void d_cat_walk(int used_bin, int max_num_cat, int num_data, double sum_h, double cnt_factor, const SplitParams& p,
                                           int rand_i, Next next, Visit visit) {
  int cnt_cur_group = 0, left_count = 0;
  double slg = 0.0, slh = kEpsD;
  for (int i = 0; i < used_bin && i < max_num_cat; ++i) {
    double g, h;
    next(&g, &h);
    const int cnt = static_cast<int>(h * cnt_factor + 0.5);
    slg += g; slh += h; left_count += cnt; cnt_cur_group += cnt;
    if (left_count < p.min_data_in_leaf || slh < p.min_sum_hessian) continue;
    const int right_count = num_data - left_count;
    if (right_count < p.min_data_in_leaf || right_count < p.min_data_per_group) break;
    const double srh = sum_h - slh;
    if (srh < p.min_sum_hessian) break;
    if (cnt_cur_group < p.min_data_per_group) continue;
    cnt_cur_group = 0;
    if (kExtra && i != rand_i) continue;
    visit(i, slg, slh, srh, left_count);
  }
}

// Categorical split search for one feature by one warp (FeatureHistogram::FindBestThresholdCategoricalInner [UPSTREAM]):
// one-hot when num_bin <= max_cat_to_onehot; otherwise the bins holding >= cat_smooth rows are ranked by g/(h+cat_smooth)
// (stable, ties by bin) and accumulated from both ends, at most max_cat_threshold bins, lambda_l2 += cat_l2.
// ws = this warp's shared scratch: g[256], h[256], ctr[256] doubles + order[256] + used[256] bytes.
// kExtra (extra_trees): xr is the feature's stream state before this scan's draw.  One-hot draws r over the num_bin - 1 category bins
// and evaluates only bin r + 1; many-vs-many draws r over d_cat_rand_range and evaluates only the prefixes of r + 1 bins.  Returns the
// number of draws taken (0 or 1), in every lane.
// kMono (monotone constraints or path smoothing): every gain is d_mono_split_gain's at outputs smoothed toward the leaf's output and
// clamped to the leaf's bounds, with the children's estimated counts (one-hot: num_data - cnt and cnt); categorical features carry no
// constraint of their own.  min_gain_shift is d_smooth_leaf_gain's.
template <bool kExtra, bool kMono>
__device__ __noinline__ int d_scan_feature_cat(const long long (&qg)[8], const long long (&qh)[8], int lane, const FeatMeta m, const LeafState& L,
                                                  double inv_g, double inv_h, const SplitParams& p, uint8_t* flag, SplitCand* outp, double* ws,
                                                  unsigned xr) {
  SplitCand& out = *outp;
  double* sg = ws; double* sh = ws + 256; double* sc = ws + 512;
  unsigned char* order = reinterpret_cast<unsigned char*>(ws + 768);
  const double sum_g = L.sum_g, sum_h = L.sum_h + 2 * kEpsD;
  const int num_data = L.global_count;
  const double cnt_factor = num_data / sum_h;
  const double min_gain_shift = (kMono ? d_smooth_leaf_gain(sum_g, sum_h, num_data, L.output, p) : d_leaf_gain(sum_g, sum_h, p)) + p.min_gain_to_split;
  const bool onehot = m.num_bin <= p.max_cat_to_onehot;
  int drew = 0, rand_t = -1;      // rand_t: the one candidate index evaluated, -1: every candidate
  if (kExtra && onehot) { rand_t = d_extra_draw(&xr, m.num_bin - 1); drew = m.num_bin > 1 ? 1 : 0; }
  bool any_valid = false;
  double best_gain = kNegInf, best_lg = 0, best_lh = 0;
  int best_t = 0x7fffffff, best_lc = 0;
  unsigned used_mask = 0;      // bit j: my bin j is "used" (enough rows)
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int b = lane * 8 + j;
    const double g = static_cast<double>(qg[j]) * inv_g, h = static_cast<double>(qh[j]) * inv_h;
    sg[b] = g; sh[b] = h;
    const int cnt = static_cast<int>(h * cnt_factor + 0.5);
    const bool in_range = b >= 1 && b < m.num_bin;
    if (onehot) {
      if (in_range && !(cnt < p.min_data_in_leaf || h < p.min_sum_hessian)) {
        const int other = num_data - cnt;
        const double oh = sum_h - h - kEpsD;
        if (other >= p.min_data_in_leaf && oh >= p.min_sum_hessian && (!kExtra || b - 1 == rand_t)) {
          const double gain = kMono ? d_mono_split_gain(sum_g - g, oh, g, h + kEpsD, other, cnt, L.output, p, L.mono_min, L.mono_max, 0)
                                    : d_leaf_gain(sum_g - g, oh, p) + d_leaf_gain(g, h + kEpsD, p);
          if (gain > min_gain_shift) {
            any_valid = true;
            if (gain > best_gain) { best_gain = gain; best_t = b; best_lg = g; best_lh = h + kEpsD; best_lc = cnt; }
          }
        }
      }
    } else {
      const bool used = in_range && cnt >= p.cat_smooth;
      if (used) used_mask |= 1u << j;
      sc[b] = g / (h + p.cat_smooth);
    }
  }
  __syncwarp();
  if (onehot) {
    for (int o = 16; o; o >>= 1) {        // first seen = smallest bin wins ties
      const double og = __shfl_xor_sync(0xffffffffu, best_gain, o);
      const int ot = __shfl_xor_sync(0xffffffffu, best_t, o), oc = __shfl_xor_sync(0xffffffffu, best_lc, o);
      const double olg = __shfl_xor_sync(0xffffffffu, best_lg, o), olh = __shfl_xor_sync(0xffffffffu, best_lh, o);
      if (og > best_gain || (og == best_gain && ot < best_t)) { best_gain = og; best_t = ot; best_lg = olg; best_lh = olh; best_lc = oc; }
    }
    any_valid = __any_sync(0xffffffffu, any_valid);
    if (lane == 0) {
      *flag = any_valid ? 1 : 0;
      if (any_valid) {
        out.gain = best_gain - min_gain_shift; out.left_g = best_lg; out.left_h = best_lh; out.threshold = 0; out.left_count = best_lc;
        out.default_left = 0; out.is_cat = 1; out.l2_extra = 0;
        out.cat_bits[best_t >> 5] |= 1u << (best_t & 31);
      }
    }
    return drew;
  }
  // ---- rank the used bins by ctr (stable): rank = #{used j : ctr_j < ctr_i  or (== and j < i)}.
  // Uniform loop over the bins: sc[bj] / usedb[bj] are broadcast loads, the 8 comparisons of a lane are independent.
  unsigned char* usedb = order + 256;
  int used_bin = 0;
  double ci[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int b = lane * 8 + j;
    const bool u = (used_mask >> j) & 1u;
    usedb[b] = u ? 1 : 0;
    ci[j] = sc[b];
    used_bin += __popc(__ballot_sync(0xffffffffu, u));
  }
  if (kExtra) {
    const int range = d_cat_rand_range(used_bin, p.max_cat_threshold);
    rand_t = d_extra_draw(&xr, range);
    drew = range > 0 ? 1 : 0;
  }
  __syncwarp();
  int rank[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) rank[j] = 0;
  for (int bj = 1; bj < m.num_bin; ++bj) {
    if (!usedb[bj]) continue;             // same bj in every lane: no divergence
    const double cj = sc[bj];
#pragma unroll
    for (int j = 0; j < 8; ++j) rank[j] += (cj < ci[j]) || (cj == ci[j] && bj < lane * 8 + j);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if ((used_mask >> j) & 1u) order[rank[j]] = static_cast<unsigned char>(lane * 8 + j);
  __syncwarp();
  if (lane == 0) {
    SplitParams pc = p;
    pc.l2 += p.cat_l2;
    const int max_num_cat = min(p.max_cat_threshold, (used_bin + 1) / 2);
    int best_i = -1, best_dir = 1;
    for (int d = 0; d < 2; ++d) {
      const int dir = d == 0 ? 1 : -1;
      int pos = d == 0 ? 0 : used_bin - 1;
      d_cat_walk<kExtra>(used_bin, max_num_cat, num_data, sum_h, cnt_factor, p, rand_t,
                         [&](double* g, double* h) { const int t = order[pos]; pos += dir; *g = sg[t]; *h = sh[t]; },
                         [&](int i, double slg, double slh, double srh, int left_count) {
                           const double gain = kMono ? d_mono_split_gain(slg, slh, sum_g - slg, srh, left_count, num_data - left_count, L.output, pc,
                                                                         L.mono_min, L.mono_max, 0)
                                                     : d_leaf_gain(slg, slh, pc) + d_leaf_gain(sum_g - slg, srh, pc);
                           if (gain <= min_gain_shift) return;
                           any_valid = true;
                           if (gain > best_gain) { best_gain = gain; best_lg = slg; best_lh = slh; best_lc = left_count; best_i = i; best_dir = dir; }
                         });
    }
    *flag = any_valid ? 1 : 0;
    if (any_valid) {
      out.gain = best_gain - min_gain_shift; out.left_g = best_lg; out.left_h = best_lh; out.threshold = 0; out.left_count = best_lc;
      out.default_left = 0; out.is_cat = 1; out.l2_extra = p.cat_l2;
      for (int i = 0; i <= best_i; ++i) {
        const int t = best_dir == 1 ? order[i] : order[used_bin - 1 - i];
        out.cat_bits[t >> 5] |= 1u << (t & 31);
      }
    }
  }
  return drew;
}

// forced_leaf >= 0: the forced phase splits that leaf (its best is the plan node's split) instead of the arg-max
__device__ __forceinline__ void d_choose_leaf(TreeCtrl* ctrl, LeafState* leaves, const FeatMeta* __restrict__ meta, const SplitParams& p, int lane,
                                              int forced_leaf) {
  double bg = kNegInf; int bf = 0x7fffffff, bl = 0x7fffffff;
  const int nl = ctrl->num_leaves;
  for (int l = lane; l < nl; l += 32) {
    const double g = leaves[l].best.gain;
    const int fi = leaves[l].best.feature;
    const int f = fi < 0 ? 0x7fffffff : meta[fi].real_index;
    if (g > bg || (g == bg && (f < bf || (f == bf && l < bl)))) { bg = g; bf = f; bl = l; }
  }
  for (int o = 16; o; o >>= 1) {
    const double og = __shfl_xor_sync(0xffffffffu, bg, o);
    const int of = __shfl_xor_sync(0xffffffffu, bf, o), ol = __shfl_xor_sync(0xffffffffu, bl, o);
    if (og > bg || (og == bg && (of < bf || (of == bf && ol < bl)))) { bg = og; bf = of; bl = ol; }
  }
  if (lane != 0) return;
  const int best_leaf = forced_leaf >= 0 ? forced_leaf : (bl == 0x7fffffff ? 0 : bl);
  const LeafBest& b = leaves[best_leaf].best;
  if (!(b.gain > 0.0) || ctrl->num_leaves >= p.num_leaves) {
    ctrl->finished = 1; ctrl->split_leaf = -1; ctrl->part_count = 0;
  } else {
    const LeafState& L = leaves[best_leaf];
    const FeatMeta fm = meta[b.feature];
    ctrl->split_leaf = best_leaf; ctrl->new_leaf = ctrl->num_leaves; ctrl->pending = 1;
    ctrl->split_feature = b.feature; ctrl->split_threshold = b.threshold; ctrl->split_default_left = b.default_left;
    ctrl->split_missing_type = fm.missing_type; ctrl->split_num_bin = fm.num_bin;
    ctrl->split_is_cat = b.is_cat;
    for (int wd = 0; wd < 8; ++wd) ctrl->split_cat_bits[wd] = b.cat_bits[wd];
    ctrl->split_wide = b.feature >= p.nfn ? b.feature - p.nfn : -1;
    ctrl->split_cat_list_len = b.cat_list_len;
    for (int k = 0; k < b.cat_list_len && k < kCatListMax; ++k) ctrl->split_cat_list[k] = b.cat_list[k];
    ctrl->part_begin = L.begin; ctrl->part_count = L.count; ctrl->part_buf = L.buf; ctrl->part_identity = L.identity;
    ctrl->part_left_total = 0;
  }
}

// candidates are written by other blocks of the same kernel: read them through L2 (ld.global.cg), never from this SM's L1
__device__ __forceinline__ SplitCand d_load_cand(const SplitCand* c) {
  static_assert(sizeof(SplitCand) % 8 == 0, "SplitCand is copied in 8-byte words");
  SplitCand out;
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(c);
  unsigned long long* dst = reinterpret_cast<unsigned long long*>(&out);
#pragma unroll
  for (int i = 0; i < static_cast<int>(sizeof(SplitCand) / 8); ++i) dst[i] = __ldcg(src + i);
  return out;
}
// a leaf's best split from its candidate c ([UPSTREAM] SplitInfo as FindBestThreshold leaves it): sums without the scans' epsilon, the
// children's outputs (kMono: smoothed toward the leaf's output and clamped to its bounds) and what the round controller's constraint
// update needs
template <bool kMono>
__device__ __forceinline__ void d_leaf_best(const SplitCand& c, const LeafState& L, const SplitParams& p, const signed char* __restrict__ mono_type,
                                            const unsigned long long* __restrict__ sets_of, LeafBest* out) {
  LeafBest& b = *out;
  b.monotone_type = 0; b.inter_sets = 0ull;
  b.cat_list_len = c.cat_list_len;
  for (int k = 0; k < c.cat_list_len && k < kCatListMax; ++k) b.cat_list[k] = c.cat_list[k];
  const double sum_h = L.sum_h + 2 * kEpsD;
  b.gain = c.gain; b.feature = c.feature; b.threshold = c.threshold; b.default_left = c.default_left;
  b.left_count = c.left_count; b.right_count = L.global_count - c.left_count;
  b.left_g = c.left_g; b.left_h = c.left_h - kEpsD;
  b.right_g = L.sum_g - c.left_g; b.right_h = sum_h - c.left_h - kEpsD;
  SplitParams pc = p;
  pc.l2 += c.l2_extra;
  if constexpr (kMono) {
    b.left_out = d_mono_output(c.left_g, c.left_h, b.left_count, L.output, pc, L.mono_min, L.mono_max);
    b.right_out = d_mono_output(L.sum_g - c.left_g, sum_h - c.left_h, b.right_count, L.output, pc, L.mono_min, L.mono_max);
    b.monotone_type = mono_type[c.feature];
  } else {
    b.left_out = d_calc_output(c.left_g, c.left_h, pc);
    b.right_out = d_calc_output(L.sum_g - c.left_g, sum_h - c.left_h, pc);
  }
  if (p.interaction) b.inter_sets = sets_of[c.feature];
  b.is_cat = c.is_cat;
  for (int wd = 0; wd < 8; ++wd) b.cat_bits[wd] = c.cat_bits[wd];
}

// Forced splits, the pick step's thread 0 once every leaf's best is in place ([UPSTREAM] the queue loop of SerialTreeLearner::ForceSplits):
// while the phase lasts, plan node j = forced_next splits its leaf when its stored evaluation is valid; that leaf's best becomes the
// node's split and the leaf is returned.  Otherwise (the node is invalid or was never evaluated, the plan has run out, or the tree is
// full) the phase ends and this round picks as it would without a plan (-1).  The leaf being split loses its own best split, which
// the round controller resets anyway.
template <bool kMono>
__device__ __noinline__ int d_forced_pick(TreeCtrl* ctrl, LeafState* leaves, const ForcedArgs& forced, const SplitParams& p,
                                          const signed char* __restrict__ mono_type, const unsigned long long* __restrict__ sets_of) {
  const int j = ctrl->forced_next;
  if (j < 0 || ctrl->finished) return -1;
  if (j < forced.n && ctrl->num_leaves < p.num_leaves) {
    const SplitCand c = d_load_cand(&forced.evals[j]);
    if (c.gain > 0.0) {
      const int leaf = forced.nodes[j].leaf;
      d_leaf_best<kMono>(c, leaves[leaf], p, mono_type, sets_of, &leaves[leaf].best);
      ctrl->forced_next = j + 1;
      return leaf;
    }
  }
  ctrl->forced_next = -1;
  return -1;
}

// best candidate per leaf (argmax over features, ties -> smaller real feature index), then the leaf to split; one 256-thread block.
// The two leaves of the round are handled side by side (threads 0..127: smaller, 128..255: larger) with warp-shuffle argmaxes — the
// first version looped over the two leaves with an 8-step shared-memory tree each (18 block barriers) and ncu showed this serial tail
// taking longer than the scan itself.  The order (gain desc, real feature index asc) is total, so any reduction shape picks the same winner.
// kMono (monotone constraints or path smoothing): the outputs are smoothed toward the leaf's output with the candidate's estimated
// counts, then clamped to the leaf's bounds ([UPSTREAM] CalculateSplittedLeafOutput<USE_MC, USE_SMOOTHING>), and the split feature's
// constraint (mono_type, per inner feature) is kept for the round controller's bound update.
// p.interaction (interaction constraints): a feature that may not split the leaf (sets_of[u] & the leaf's inter_mask == 0) is passed
// over here and only here, after the scans, so the scans, their is_splittable flags and the extra_trees draws are what they are
// without constraints ([UPSTREAM] SerialTreeLearner::ComputeBestSplitForFeature filters after FindBestThreshold).  The chosen
// feature's sets_of word is kept for the round controller's mask update.
// node_mask non-null (per-node feature sampling): likewise a feature the leaf did not sample (written by d_bynode_sample in this kernel)
// is passed over, and the ColSampler stream moves past the round's draws.
// forced.nodes non-null (forced splits): while the forced phase lasts, the next plan node's stored evaluation replaces the arg-max when it
// is valid (d_forced_pick).
template <bool kMono>
__device__ __noinline__ void
d_pick_block(TreeCtrl* ctrl, LeafState* leaves, const FeatMeta* __restrict__ meta, const SplitCand* cands, const SplitParams& p,
             const signed char* __restrict__ mono_type, const unsigned long long* __restrict__ sets_of, const uint8_t* node_mask,
             const ForcedArgs& forced) {
  __shared__ double s_gain[8];
  __shared__ int s_feat[8], s_idx[8];
  const int which = threadIdx.x >> 7, t = threadIdx.x & 127, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int leaf = ctrl->go ? (which ? ctrl->larger : ctrl->smaller) : -1;
  double bg = kNegInf; int bf = 0x7fffffff, bi = -1;
  if (leaf >= 0) {
    const unsigned long long mask = p.interaction ? leaves[leaf].inter_mask : 0ull;
    for (int u = t; u < p.nf; u += 128) {
      if (p.interaction && !(sets_of[u] & mask)) continue;
      if (node_mask && !__ldcg(&node_mask[which * p.nf_pad + u])) continue;
      const double cg = __ldcg(&cands[which * p.nf_pad + u].gain);
      const int rf = meta[u].real_index;
      if (cg > bg || (cg == bg && rf < bf)) { bg = cg; bf = rf; bi = u; }
    }
  }
  for (int o = 16; o; o >>= 1) {
    const double og = __shfl_xor_sync(0xffffffffu, bg, o);
    const int of = __shfl_xor_sync(0xffffffffu, bf, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (og > bg || (og == bg && of < bf)) { bg = og; bf = of; bi = oi; }
  }
  if (lane == 0) { s_gain[warp] = bg; s_feat[warp] = bf; s_idx[warp] = bi; }
  __syncthreads();
  if (t == 0 && leaf >= 0) {
    for (int w = which * 4; w < which * 4 + 4; ++w)
      if (s_gain[w] > bg || (s_gain[w] == bg && s_feat[w] < bf)) { bg = s_gain[w]; bf = s_feat[w]; bi = s_idx[w]; }
    LeafState& L = leaves[leaf];
    LeafBest b;
    b.gain = kNegInf; b.feature = -1; b.threshold = 0; b.default_left = 1; b.left_count = 0; b.right_count = 0;
    b.left_g = b.left_h = b.right_g = b.right_h = b.left_out = b.right_out = 0; b.is_cat = 0; b.cat_list_len = 0; b.monotone_type = 0;
    b.inter_sets = 0ull;
    for (int wd = 0; wd < 8; ++wd) b.cat_bits[wd] = 0u;
    if (bi >= 0 && bg > kNegInf) d_leaf_best<kMono>(d_load_cand(&cands[which * p.nf_pad + bi]), L, p, mono_type, sets_of, &b);
    L.best = b;
  }
  if (node_mask && threadIdx.x == 0 && ctrl->go) ctrl->col_state = __ldcg(&ctrl->col_next);
  __syncthreads();
  int forced_leaf = -1;
  if (forced.nodes) {      // the same in every thread: a kernel argument
    __shared__ int s_forced_leaf;
    if (threadIdx.x == 0) s_forced_leaf = d_forced_pick<kMono>(ctrl, leaves, forced, p, mono_type, sets_of);
    __syncthreads();
    forced_leaf = s_forced_leaf;
  }
  if (threadIdx.x < 32 && !ctrl->finished) d_choose_leaf(ctrl, leaves, meta, p, threadIdx.x, forced_leaf);
}

// ---------------------------------------------------------------- same-device all-reduce (rank-threads of one process on one device)
// Every rank's buffer is on this device, so one launch, enqueued by the last rank to reach the collective (engine.cu SameDeviceComm), does
// the whole all-reduce: element i of every buffer becomes Op over the R buffers' element i, accumulated in rank order.  The order never
// changes, so double sums are deterministic; for R = 2 they equal NCCL's a + b bit for bit.  Each thread owns whole 16-byte vectors (the
// per-split C2 histogram is 1-2 MB of int64), so reading and then overwriting all R copies in place needs no barrier.  The rank loops are
// unrolled to kMaxPeers with a guard, so the pointer table stays in the parameter bank instead of a local copy.
constexpr int kMaxPeers = 16;      // ranks that may share one device (DecideLayout)
struct SameDevicePtrs { void* p[kMaxPeers]; };
template <typename T> struct RedSum { __device__ __forceinline__ static T f(T a, T b) { return a + b; } };
template <typename T> struct RedMax { __device__ __forceinline__ static T f(T a, T b) { return b > a ? b : a; } };
template <typename T> struct RedMin { __device__ __forceinline__ static T f(T a, T b) { return b < a ? b : a; } };
// fmax / fmin for doubles (the host values reduced this way are never NaN): the compare-and-select form spills at -O3
template <> struct RedMax<double> { __device__ __forceinline__ static double f(double a, double b) { return fmax(a, b); } };
template <> struct RedMin<double> { __device__ __forceinline__ static double f(double a, double b) { return fmin(a, b); } };
template <typename T> struct alignas(16) Vec16 { T v[16 / sizeof(T)]; };

// vec: every buffer is 16-byte aligned, so count / (16 / sizeof(T)) vectors go as 16-byte loads and stores and the rest as scalars
template <typename T, typename Op>
__global__ void __launch_bounds__(256)
k_allreduce_same_device(SameDevicePtrs bufs, int R, long long count, int vec) {
  constexpr int V = 16 / sizeof(T);
  const long long nvec = vec ? count / V : 0;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (long long i = tid; i < nvec; i += stride) {
    Vec16<T> acc = reinterpret_cast<const Vec16<T>*>(bufs.p[0])[i];
#pragma unroll
    for (int r = 1; r < kMaxPeers; ++r) {
      if (r < R) {
        const Vec16<T> x = reinterpret_cast<const Vec16<T>*>(bufs.p[r])[i];
#pragma unroll
        for (int k = 0; k < V; ++k) acc.v[k] = Op::f(acc.v[k], x.v[k]);
      }
    }
#pragma unroll
    for (int r = 0; r < kMaxPeers; ++r)
      if (r < R) reinterpret_cast<Vec16<T>*>(bufs.p[r])[i] = acc;
  }
  for (long long i = nvec * V + tid; i < count; i += stride) {
    T acc = static_cast<const T*>(bufs.p[0])[i];
#pragma unroll
    for (int r = 1; r < kMaxPeers; ++r)
      if (r < R) acc = Op::f(acc, static_cast<const T*>(bufs.p[r])[i]);
#pragma unroll
    for (int r = 0; r < kMaxPeers; ++r)
      if (r < R) static_cast<T*>(bufs.p[r])[i] = acc;
  }
}

// ---------------------------------------------------------------- column-major copy of the uint8 tiles (for the partition kernel)
// The tile layout [tile][row][32 features] is what K4 streams, but the partition kernel needs ONE feature of every row of a leaf and pays
// a 32-byte sector for each byte (62 % of its DRAM bytes at 100M rows).  When device memory allows, the booster keeps a second copy
// [feature][row] (cols_stride = rows rounded up to 256), built once by this kernel.
__global__ void __launch_bounds__(256)
k_tiles_to_columns(const uint8_t* __restrict__ bins, size_t rows_stride, int num_tiles, long long nrow, uint8_t* __restrict__ cols, size_t cols_stride) {
  __shared__ uint4 s_t[256 * 2 + 16];                      // 256 rows x 32 bytes
  const long long per_tile = (nrow + 255) / 256;
  for (long long w = blockIdx.x; w < per_tile * num_tiles; w += gridDim.x) {
    const int tile = static_cast<int>(w / per_tile);
    const long long r0 = (w % per_tile) * 256;
    const int rows = static_cast<int>(min(256LL, nrow - r0));
    const uint4* src = reinterpret_cast<const uint4*>(bins + (static_cast<size_t>(tile) * rows_stride + static_cast<size_t>(r0)) * 32);
    __syncthreads();
    for (int i = threadIdx.x; i < rows * 2; i += 256) s_t[i] = src[i];
    __syncthreads();
    const uint8_t* sb = reinterpret_cast<const uint8_t*>(s_t);
    const int f = threadIdx.x >> 3, g = threadIdx.x & 7;   // feature of the tile, group of 32 rows
    unsigned wv[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      unsigned v = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) { const int r = g * 32 + k * 4 + j; v |= (r < rows ? static_cast<unsigned>(sb[r * 32 + f]) : 0u) << (8 * j); }
      wv[k] = v;
    }
    uint4* dst = reinterpret_cast<uint4*>(cols + (static_cast<size_t>(tile) * 32 + f) * cols_stride + static_cast<size_t>(r0) + g * 32);
    dst[0] = make_uint4(wv[0], wv[1], wv[2], wv[3]);       // cols_stride is a multiple of 256: padding rows exist and are never read
    dst[1] = make_uint4(wv[4], wv[5], wv[6], wv[7]);
  }
}

// When the whole copy does not fit, the booster keeps a pool of column slots instead and fills them, between trees, with the storage
// columns the trees split on (TreeLearner::UpdateColumnCache).  This kernel copies up to kColumnBuildsMax storage columns into given slots:
// blockIdx.y is the job, each thread packs 4 consecutive rows into one 32-bit store.  The 4 bytes lie in 4 sectors of one 128-byte
// line, so every sector of the column's tile is read from DRAM once per job (32 bytes per row).
constexpr int kColumnBuildsMax = 8;
struct ColumnJobs { int n; int col[kColumnBuildsMax]; int slot[kColumnBuildsMax]; };
__global__ void __launch_bounds__(256)
k_tiles_to_column_slots(const uint8_t* __restrict__ bins, size_t rows_stride, long long nrow, ColumnJobs jobs, uint8_t* __restrict__ cols,
                        size_t cols_stride) {
  const int c = jobs.col[blockIdx.y];
  const uint8_t* src = bins + static_cast<size_t>(c >> 5) * rows_stride * 32 + (c & 31);
  unsigned* dst = reinterpret_cast<unsigned*>(cols + static_cast<size_t>(jobs.slot[blockIdx.y]) * cols_stride);     // cols_stride: multiple of 256
  const long long words = (nrow + 3) / 4;
  for (long long w = blockIdx.x * 256LL + threadIdx.x; w < words; w += static_cast<long long>(gridDim.x) * 256) {
    const long long r0 = w * 4;
    unsigned v = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (r0 + j < nrow) v |= static_cast<unsigned>(src[static_cast<size_t>(r0 + j) * 32]) << (8 * j);
    dst[w] = v;
  }
}

// ---------------------------------------------------------------- K7 row partition (stable), one cooperative kernel per split
// Replaces [UPSTREAM] DataPartition::Split.  Round 1 ran three kernels (decision bits + per-chunk left counts, single-block scan of the
// chunk counts, scatter) plus a memset of the scratch histogram and the next round's controller: five launches on the per-split
// critical path.  They are now the phases of ONE cooperatively launched kernel separated by software grid barriers (all blocks are
// resident; the arrive counter lives in TreeCtrl):
//   phase 0  zero the scratch histogram H for the next K4 (the scan kernel consumed it; stream order)
//   phase 1  decision bit per row (ballot words) and the left count of every 2048-row chunk
//   ---- grid barrier
//   phase 2  chunk prefix: leaves of <= 2048 chunks (4M rows) are scanned redundantly by every block in shared memory (no second
//            barrier); larger ones in two levels (one block per 2048 counts, second barrier, every block scans the totals)
//   phase 3  stable scatter into the other index buffer (lefts first, then rights, original order kept); the (g,h) words of the
//            child K4 scans next go into partition order (qord)
//   tail     the block that finishes last applies the split to the tree and prepares the next round (d_round_ctl)
constexpr int kPartChunk = 2048;     // rows per chunk = 256 threads x 8
constexpr int kPartLocalScan = 2048; // chunk counts a block scans by itself
__device__ __forceinline__ bool d_goes_left(unsigned bin, const TreeCtrl* c) {
  if (c->split_is_cat) return (c->split_cat_bits[bin >> 5] >> (bin & 31u)) & 1u;
  if (c->split_missing_type == 2 && bin == static_cast<unsigned>(c->split_num_bin - 1)) return c->split_default_left != 0;
  return bin <= static_cast<unsigned>(c->split_threshold);
}
// all blocks of a cooperative launch: arrive on a monotone counter, spin until `target` arrivals
__device__ __forceinline__ void d_grid_barrier(unsigned* counter, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    while (*reinterpret_cast<volatile unsigned*>(counter) < target) __nanosleep(32);
    __threadfence();
  }
  __syncthreads();
}
__global__ void __launch_bounds__(256, 3)
k_partition(TreeCtrl* ctrl, LeafState* leaves, TreeDev tree, uint8_t* flags, const FeatMeta* __restrict__ meta, SplitParams p, int last,
            const uint8_t* __restrict__ bins, size_t rows_stride, int* __restrict__ idx0, int* __restrict__ idx1, unsigned* __restrict__ bits,
            int* __restrict__ chunk_left, const int4* __restrict__ qgh, int4* __restrict__ qord, long long* __restrict__ H, size_t h_elems,
            const uint16_t* __restrict__ bins16, int tickets_per_block, const uint8_t* __restrict__ cols, size_t cols_stride,
            const int* __restrict__ col_slot, int* __restrict__ super_tot, const int* __restrict__ bundle_base) {
  __shared__ int s_pref[kPartLocalScan + 1];
  __shared__ unsigned short s_list[kCatListMax];
  __shared__ int s_wl[64];
  __shared__ int s_cnt[8];
  __shared__ int s_copy[2];
  __shared__ int s_last;
  __shared__ int s_chunk;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // ---- phase 0: H := 0 (16-byte stores; H is L2-resident)
  {
    longlong2* h2 = reinterpret_cast<longlong2*>(H);
    const size_t n2 = h_elems / 2;
    const longlong2 z = make_longlong2(0, 0);
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n2; i += static_cast<size_t>(gridDim.x) * blockDim.x) h2[i] = z;
  }
  const int n = ctrl->part_count;
  if (n > 0) {
    const int* src = ctrl->part_buf ? idx1 : idx0;
    int* dst = ctrl->part_identity ? idx0 : (ctrl->part_buf ? idx0 : idx1);
    const int begin = ctrl->part_begin, identity = ctrl->part_identity;
    const int f = ctrl->split_feature;
    const int wide = ctrl->split_wide;
    const int sc = wide >= 0 ? 0 : meta[f].hist_off >> 8;         // storage column of the split feature
    const int bbase = (wide >= 0 || !bundle_base) ? -1 : bundle_base[f], bmfb = meta[f].default_bin, bnb = meta[f].num_bin;
    const uint8_t* col = bins + (static_cast<size_t>(sc >> 5) * rows_stride) * 32 + (sc & 31);
    const uint16_t* wcol = wide >= 0 ? bins16 + static_cast<size_t>(wide) * rows_stride : nullptr;
    // column-major copy of the split's storage column, if the booster keeps one: col_slot maps a storage column to its slot (-1: none)
    const int cslot = (col_slot != nullptr && wide < 0) ? col_slot[sc] : -1;
    const uint8_t* ccol = cslot >= 0 ? cols + static_cast<size_t>(cslot) * cols_stride : nullptr;
    const bool wide_cat = wide >= 0 && ctrl->split_is_cat;
    const int list_len = wide_cat ? ctrl->split_cat_list_len : 0;
    if (threadIdx.x < list_len) s_list[threadIdx.x] = ctrl->split_cat_list[threadIdx.x];
    __syncthreads();
    const int chunks = (n + kPartChunk - 1) / kPartChunk;
    // ---- phase 1 (no block-wide barrier: every warp adds the left count of its 256 rows to the chunk's counter, which the tail of
    // the previous partition kernel left at zero)
    // chunks are handed out dynamically (one atomic per chunk): the rows' DRAM latency varies, and the grid barrier waits for the slowest block
    // a ticket grants `grp` consecutive chunks: a 100M-row leaf has 48K chunks, and one same-address atomic per chunk and phase is a
    // serial ~100 us; with ~tickets_per_block tickets per block the hand-out stays dynamic and the atomics are negligible
    const int grp = tickets_per_block > 0 ? max(1, chunks / (static_cast<int>(gridDim.x) * tickets_per_block)) : 1;
    for (;;) {
      __syncthreads();
      if (threadIdx.x == 0) s_chunk = static_cast<int>(atomicAdd(&ctrl->part_next[0], 1u));
      __syncthreads();
      const int cbase = s_chunk * grp;
      if (cbase >= chunks) break;
      for (int c = cbase; c < min(cbase + grp, chunks); ++c) {
      // the 8 rows of a thread: all index loads first, then all bin loads, then the ballots — two dependent memory latencies per chunk
      // instead of sixteen (ncu, 100M-row table: the kernel ran at 2 TB/s with long_scoreboard as the only stall reason)
      int local = 0;
      int rr[8]; unsigned bb[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int i = c * kPartChunk + k * 256 + threadIdx.x;
        rr[k] = i < n ? (identity ? (begin + i) : src[begin + i]) : -1;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        bb[k] = 0u;
        if (rr[k] >= 0)
          bb[k] = wide >= 0 ? static_cast<unsigned>(wcol[rr[k]]) : (ccol ? static_cast<unsigned>(ccol[rr[k]]) : static_cast<unsigned>(col[static_cast<size_t>(rr[k]) * 32]));
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        bool left = false;
        if (rr[k] >= 0) {
          const unsigned bin = d_unbundle(bb[k], bbase, bmfb, bnb);
          if (wide_cat) { for (int kk = 0; kk < list_len; ++kk) left |= (bin == s_list[kk]); }
          else left = d_goes_left(bin, ctrl);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, left);
        if (lane == 0) { bits[(c * kPartChunk + k * 256 + threadIdx.x) >> 5] = bal; local += __popc(bal); }
      }
      if (lane == 0 && local) atomicAdd(&chunk_left[c], local);
      }
    }
    d_grid_barrier(&ctrl->part_barrier, gridDim.x);
    // ---- phase 2: exclusive prefix of the chunk counts + total
    int total_left;
    const bool local_scan = chunks <= kPartLocalScan;
    if (local_scan) {
      // 256 threads x 8 consecutive counts, warp scan of the per-thread sums, then the block total
      int v[8], sum = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) { const int i = threadIdx.x * 8 + k; v[k] = i < chunks ? __ldcg(chunk_left + i) : 0; sum += v[k]; }
      int inc = sum;
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      if (lane == 31) s_cnt[warp] = inc;
      __syncthreads();
      int woff = 0;
      for (int w = 0; w < warp; ++w) woff += s_cnt[w];
      int run = woff + inc - sum;
#pragma unroll
      for (int k = 0; k < 8; ++k) { s_pref[threadIdx.x * 8 + k] = run; run += v[k]; }
      if (threadIdx.x == 255) s_pref[kPartLocalScan] = run;
      __syncthreads();
      total_left = s_pref[kPartLocalScan];
    } else {
      // two levels: block s scans the 2048 counts of "super-chunk" s in place (prefix relative to the super-chunk) and publishes its total;
      // after the second barrier every block scans the totals.  (The first version had block 0 scan all counts alone: ~190 us for the 48K
      // chunks of a 100M-row root while every other block waited at the barrier.)
      const int supers = (chunks + kPartLocalScan - 1) / kPartLocalScan;
      for (int sp = blockIdx.x; sp < supers; sp += gridDim.x) {
        int v[8], sum = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { const int i = sp * kPartLocalScan + threadIdx.x * 8 + k; v[k] = i < chunks ? __ldcg(chunk_left + i) : 0; sum += v[k]; }
        int inc = sum;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        __syncthreads();
        if (lane == 31) s_cnt[warp] = inc;
        __syncthreads();
        int woff = 0;
        for (int w = 0; w < warp; ++w) woff += s_cnt[w];
        int run = woff + inc - sum;
#pragma unroll
        for (int k = 0; k < 8; ++k) { const int i = sp * kPartLocalScan + threadIdx.x * 8 + k; if (i < chunks) chunk_left[i] = run; run += v[k]; }
        if (threadIdx.x == 255) super_tot[sp] = run;
      }
      d_grid_barrier(&ctrl->part_barrier, 2 * gridDim.x);
      {   // exclusive scan of the super-chunk totals (at most 2048 of them: 8.6G rows) into s_pref
        int v[8], sum = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { const int i = threadIdx.x * 8 + k; v[k] = i < supers ? __ldcg(super_tot + i) : 0; sum += v[k]; }
        int inc = sum;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        __syncthreads();
        if (lane == 31) s_cnt[warp] = inc;
        __syncthreads();
        int woff = 0;
        for (int w = 0; w < warp; ++w) woff += s_cnt[w];
        int run = woff + inc - sum;
#pragma unroll
        for (int k = 0; k < 8; ++k) { s_pref[threadIdx.x * 8 + k] = run; run += v[k]; }
        if (threadIdx.x == 255) s_pref[kPartLocalScan] = run;
        __syncthreads();
        total_left = s_pref[kPartLocalScan];
      }
    }
    // the child K4 scans next is the one with fewer rows by the rule of d_round_ctl (global counts of the split in data-parallel
    // mode, true counts otherwise; ties -> right): its (g,h) words are written in partition order (qord)
    const LeafBest& bsp = leaves[ctrl->split_leaf].best;
    const int lc = p.parallel ? bsp.left_count : total_left, rc = p.parallel ? bsp.right_count : n - total_left;
    const bool q_left = lc < rc;
    // ---- phase 3
    for (;;) {
      __syncthreads();
      if (threadIdx.x == 0) s_chunk = static_cast<int>(atomicAdd(&ctrl->part_next[1], 1u));
      __syncthreads();
      const int cbase = s_chunk * grp;
      if (cbase >= chunks) break;
      for (int c = cbase; c < min(cbase + grp, chunks); ++c) {
      const int wbase = c * (kPartChunk / 32);     // 64 ballot words per chunk; word w covers rows c*2048 + w*32 ..
      if (threadIdx.x < 64) {
        const int i0 = c * kPartChunk + threadIdx.x * 32;
        s_wl[threadIdx.x] = i0 < n ? __popc(__ldcg(bits + wbase + threadIdx.x)) : 0;
      }
      __syncthreads();
      if (warp == 0) {   // exclusive scan of the 64 word counts (two per lane)
        const int a = s_wl[lane * 2], b = s_wl[lane * 2 + 1];
        const int sum = a + b;
        int inc = sum;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        const int ex = inc - sum;
        s_wl[lane * 2] = ex; s_wl[lane * 2 + 1] = ex + a;
      }
      __syncthreads();
      const int left_base = local_scan ? s_pref[c] : s_pref[c / kPartLocalScan] + __ldcg(chunk_left + c);
      const int right_base = c * kPartChunk - left_base;
      // same batching as phase 1: the 8 index loads, then the (g,h) words of the rows that go to the child K4 scans next, then the stores
      int rr[8], pp[8]; bool qq[8]; int4 qv[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int w = k * 8 + warp;                 // word index inside the chunk
        const int i = c * kPartChunk + w * 32 + lane;
        rr[k] = -1; pp[k] = 0; qq[k] = false;
        if (i < n) {
          const unsigned word = __ldcg(bits + wbase + w);
          const bool left = (word >> lane) & 1u;
          const int lefts_before = s_wl[w] + __popc(word & ((1u << lane) - 1u));
          rr[k] = identity ? (begin + i) : src[begin + i];
          pp[k] = left ? begin + left_base + lefts_before : begin + total_left + right_base + (w * 32 + lane - lefts_before);
          qq[k] = (left == q_left);
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) if (qq[k]) qv[k] = qgh[rr[k]];      // replaces a separate gather pass before K4 (k_gather_q)
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (rr[k] < 0) continue;
        dst[pp[k]] = rr[k];
        if (qq[k]) qord[pp[k]] = qv[k];
      }
      __syncthreads();      // s_wl is rewritten for the next chunk
      }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) ctrl->part_left_total = total_left;
  }
  // ---- tail: the last block to finish runs the controller of the next round
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned t = atomicAdd(&ctrl->part_ticket, 1u);
    s_last = (t == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    if (threadIdx.x == 0) { ctrl->part_ticket = 0u; ctrl->part_barrier = 0u; ctrl->part_next[0] = 0u; ctrl->part_next[1] = 0u; }
    if (n > 0) for (int c = threadIdx.x; c < (n + kPartChunk - 1) / kPartChunk; c += blockDim.x) chunk_left[c] = 0;      // phase 1 of the next launch accumulates into zeros
    d_round_ctl(ctrl, leaves, tree, flags, meta, p, last, s_copy);
  }
}

// ---------------------------------------------------------------- wide features (> 256 bins): binning, histogram, categorical scan
// value -> bin of the wide columns of a row block; wmeta = meta + nfn, the wide features' descriptions
template <typename T>
__global__ void k_bin_wide(const T* __restrict__ X, long long nrow, int row_major, long long ld, const FeatMeta* __restrict__ wmeta, int nw,
                           const double* __restrict__ ub, const uint16_t* __restrict__ catbin, uint16_t* __restrict__ bins16, size_t rows_stride,
                           long long row_offset) {
  const long long total = nrow * nw;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(e / nrow);
    const long long r = e - static_cast<long long>(w) * nrow;
    const FeatMeta m = wmeta[w];
    const double v = row_major ? static_cast<double>(X[r * ld + m.real_index]) : static_cast<double>(X[static_cast<long long>(m.real_index) * ld + r]);
    bins16[static_cast<size_t>(w) * rows_stride + row_offset + r] = static_cast<uint16_t>(d_value_to_bin(v, m, ub + m.table_off, 1, catbin + m.table_off));
  }
}

// K4 for wide features.  One CTA = (wide feature, row range of the leaf): the sub-histogram is [NATOM planes][num_bin] in shared memory
// with the same fixed-point fields as the tile kernel; lanes read consecutive rows of the uint16 column (or gather through the leaf's
// index list), so the atomics of a warp fall on data-dependent banks — these features are a few percent of a wide table's columns and
// run at a fraction of the tile kernel's rate, which is acceptable.  Flush every 2^14 rows (field headroom) into the int64 histogram.
constexpr int kWideThreads = 1024;     // one CTA per SM (128 KB of planes): the loop is latency-bound, so as many rows in flight as the SM allows
template <int NATOM>
__global__ void __launch_bounds__(kWideThreads, 1)
k4_hist_wide(const uint16_t* __restrict__ bins16, size_t rows_stride, const FeatMeta* __restrict__ wmeta, const int4* __restrict__ qgh,
             const int4* __restrict__ qord, const int* __restrict__ idx0, const int* __restrict__ idx1, const HistWork* __restrict__ work,
             unsigned long long* __restrict__ hist) {
  extern __shared__ __align__(16) unsigned wplane[];        // [NATOM][nb_pad]
  const HistWork w = *work;
  const int n = w.count;
  if (n <= 0) return;
  const int active = min(static_cast<int>(gridDim.x), (n + 4095) / 4096);
  if (static_cast<int>(blockIdx.x) >= active) return;
  const FeatMeta m = wmeta[blockIdx.y];      // wmeta = meta + nfn
  const unsigned lo = blockIdx.z * kWideHistSeg;             // this CTA accumulates bins [lo, lo + nb) of the feature
  if (static_cast<int>(lo) >= m.num_bin) return;
  const int nb = min(kWideHistSeg, m.num_bin - static_cast<int>(lo));
  const int p0 = static_cast<int>(static_cast<long long>(n) * blockIdx.x / active), p1 = static_cast<int>(static_cast<long long>(n) * (blockIdx.x + 1) / active);
  const int* __restrict__ idx = w.buf ? idx1 : idx0;
  const uint16_t* __restrict__ col = bins16 + static_cast<size_t>(blockIdx.y) * rows_stride;
  unsigned* pl0 = wplane; unsigned* pl1 = wplane + kWideHistSeg; unsigned* pl2 = wplane + 2 * kWideHistSeg; unsigned* pl3 = wplane + 3 * kWideHistSeg;
  for (int e = threadIdx.x; e < nb; e += kWideThreads) { pl0[e] = 0u; pl1[e] = 0u; pl2[e] = 0u; if (NATOM == 4) pl3[e] = 0u; }
  __syncthreads();
  for (int c0 = p0; c0 < p1; c0 += kFlushRows) {
    const int c1 = min(c0 + kFlushRows, p1);
    // four rows per thread in flight (index -> bin is a dependent pair of DRAM/L2 accesses; with one CTA per SM the loop is latency-bound)
    for (int p = c0 + threadIdx.x; p < c1; p += 4 * kWideThreads) {
      int4 q[4]; unsigned b[4]; size_t r[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int pj = p + j * kWideThreads;
        r[j] = 0;
        if (pj < c1) {
          if (w.use_idx) { r[j] = static_cast<size_t>(idx[w.begin + pj]); q[j] = qord[w.begin + pj]; }
          else { r[j] = static_cast<size_t>(w.begin + pj); q[j] = qgh[r[j]]; }
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = (p + j * kWideThreads < c1) ? static_cast<unsigned>(col[r[j]]) - lo : 0xffffffffu;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (b[j] >= static_cast<unsigned>(nb)) continue;           // another segment's bin (or past the end)
        atomicAdd(&pl0[b[j]], static_cast<unsigned>(q[j].x));
        atomicAdd(&pl1[b[j]], static_cast<unsigned>(q[j].y));
        atomicAdd(&pl2[b[j]], static_cast<unsigned>(q[j].z));
        if (NATOM == 4) atomicAdd(&pl3[b[j]], static_cast<unsigned>(q[j].w));
      }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nb; e += kWideThreads) {
      const unsigned ghi = pl0[e], glo = pl1[e], hhi = pl2[e], hlo = (NATOM == 4) ? pl3[e] : 0u;
      if (ghi | glo | hhi | hlo) {
        const long long g = (static_cast<long long>(static_cast<int>(ghi)) << kLoBits) + static_cast<long long>(glo);
        const long long h = (NATOM == 4) ? (static_cast<long long>(static_cast<int>(hhi)) << kLoBits) + static_cast<long long>(hlo) : static_cast<long long>(hhi);
        const size_t o = (static_cast<size_t>(m.hist_off) + lo + e) * 2;
        if (g) atomicAdd(&hist[o], static_cast<unsigned long long>(g));
        if (h) atomicAdd(&hist[o + 1], static_cast<unsigned long long>(h));
        pl0[e] = 0u; pl1[e] = 0u; pl2[e] = 0u; if (NATOM == 4) pl3[e] = 0u;
      }
    }
    __syncthreads();
  }
}

// exclusive prefix (reverse == 0: over threads < t) or suffix (reverse == 1: over threads > t) sums of three int64 values across a 256-thread
// block, plus nothing else; sm = 3 * 8 long longs of shared scratch.  Exact integers: any association order gives the same result.
__device__ __forceinline__ void d_block_excl3(long long& a, long long& b, long long& c, int reverse, long long* sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long ia = a, ib = b, ic = c;
  for (int o = 1; o < 32; o <<= 1) {
    long long ta, tb, tc;
    if (reverse) { ta = __shfl_down_sync(0xffffffffu, ia, o); tb = __shfl_down_sync(0xffffffffu, ib, o); tc = __shfl_down_sync(0xffffffffu, ic, o); if (lane + o < 32) { ia += ta; ib += tb; ic += tc; } }
    else { ta = __shfl_up_sync(0xffffffffu, ia, o); tb = __shfl_up_sync(0xffffffffu, ib, o); tc = __shfl_up_sync(0xffffffffu, ic, o); if (lane >= o) { ia += ta; ib += tb; ic += tc; } }
  }
  __syncthreads();
  if (lane == (reverse ? 0 : 31)) { sm[warp] = ia; sm[8 + warp] = ib; sm[16 + warp] = ic; }
  __syncthreads();
  long long oa = 0, ob = 0, oc = 0;
  for (int w2 = 0; w2 < 8; ++w2) if (reverse ? w2 > warp : w2 < warp) { oa += sm[w2]; ob += sm[8 + w2]; oc += sm[16 + w2]; }
  a = oa + ia - a; b = ob + ib - b; c = oc + ic - c;
  __syncthreads();
}

// FeatureHistogram::FindBestThresholdSequentially for a numerical feature: its reverse pass and, for NaN-as-missing features, its forward
// pass, with the bins spread over a 256-thread block — thread t owns the contiguous bins [t*S, (t+1)*S) — exclusive block scans of the per-thread
// (g, h, count) sums, and a block argmax with the sequential scan's tie-breaks (reverse pass: the highest threshold wins, forward pass: the
// lowest).  hist = the leaf's reduced histogram of the feature in its pool slot.  Returns through *outp (thread 0) and *flag.
// kExtra (extra_trees): only the candidate with that threshold is evaluated, in either pass; the count and hessian tests before it
// still skip and break as they do without it ([UPSTREAM] FindBestThresholdSequentially, USE_RAND: t - 1 + offset resp. t + offset).
// kMono (monotone constraints or path smoothing): every gain, in both passes, is d_mono_split_gain's at outputs smoothed toward the
// leaf's output with the estimated counts and clamped to the leaf's bounds, 0 when they break the feature's direction `mono`;
// min_gain_shift is d_smooth_leaf_gain's: the leaf's unconstrained gain, smoothed when path smoothing is on.
template <bool kExtra, bool kMono>
__device__ __noinline__ void d_scan_numeric(const long long* __restrict__ hist, const FeatMeta m, const LeafState& L, double inv_g, double inv_h,
                                            const SplitParams& p, uint8_t* flag, SplitCand* outp, int rand_thr, int mono) {
  __shared__ long long s_sc[24];
  __shared__ double s_bg[8], s_blg[8], s_blh[8];
  __shared__ int s_bt[8], s_blc[8], s_any, s_stop[2];
  __shared__ long long s_tot[3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double sum_g = L.sum_g, sum_h = L.sum_h + 2 * kEpsD;
  const int num_data = L.global_count;
  const double cnt_factor = num_data / sum_h;
  const double min_gain_shift = (kMono ? d_smooth_leaf_gain(sum_g, sum_h, num_data, L.output, p) : d_leaf_gain(sum_g, sum_h, p)) + p.min_gain_to_split;
  const bool two_way = (m.num_bin > 2 && m.missing_type == 2);
  const int na = two_way ? 1 : 0;
  const int S = (m.num_bin + 255) / 256;
  const int b0 = threadIdx.x * S, b1 = min(b0 + S, m.num_bin);
  if (threadIdx.x == 0) { s_any = 0; s_stop[0] = -1; s_stop[1] = blockDim.x; }     // read after the barriers of d_block_excl3
  bool any_valid = false;
  // ---- reverse pass: bins hi .. 1, candidate threshold = b - 1.  Both passes end where the sequential scan breaks: at the first candidate,
  // in scan order, whose far side fails min_data_in_leaf or min_sum_hessian_in_leaf.  A thread stops its own bins there, and the threads
  // after the first breaking one in scan order drop their candidates, so these neither win nor mark the feature splittable.  With hessians
  // >= 0 nothing after a break could pass these tests anyway (counts and hessian sums are monotone); with negative hessians (custom
  // objectives) they could.
  bool stop = false;
  double best_gain = kNegInf, best_lg = 0, best_lh = 0;
  int best_thr = -1, best_lc = 0, best_dl = 1;
  {
    const int hi = m.num_bin - 1 - na;
    long long lg = 0, lh = 0, lc = 0;
    for (int b = b0; b < b1; ++b)
      if (b >= 1 && b <= hi) { const long long qh = hist[b * 2 + 1]; lg += hist[b * 2]; lh += qh; lc += static_cast<int>(static_cast<double>(qh) * inv_h * cnt_factor + 0.5); }
    long long rg = lg, rh = lh, rc = lc;
    d_block_excl3(rg, rh, rc, 1, s_sc);
    for (int b = b1 - 1; b >= b0; --b) {
      if (b < 1 || b > hi) continue;
      const long long qg = hist[b * 2], qh = hist[b * 2 + 1];
      rg += qg; rh += qh; rc += static_cast<int>(static_cast<double>(qh) * inv_h * cnt_factor + 0.5);
      const double srg = static_cast<double>(rg) * inv_g;
      const double srh = kEpsD + static_cast<double>(rh) * inv_h;
      const int right_count = static_cast<int>(rc);
      if (right_count < p.min_data_in_leaf || srh < p.min_sum_hessian) continue;
      const int left_count = num_data - right_count;
      const double slh = sum_h - srh;
      if (left_count < p.min_data_in_leaf || slh < p.min_sum_hessian) { stop = true; break; }
      if (kExtra && b - 1 != rand_thr) continue;
      const double slg = sum_g - srg;
      const double gain = kMono ? d_mono_split_gain(slg, slh, srg, srh, left_count, right_count, L.output, p, L.mono_min, L.mono_max, mono)
                                : d_leaf_gain(slg, slh, p) + d_leaf_gain(srg, srh, p);
      if (gain <= min_gain_shift) continue;
      any_valid = true;
      if (gain > best_gain) { best_gain = gain; best_lg = slg; best_lh = slh; best_thr = b - 1; best_lc = left_count; }
    }
    if (stop) atomicMax(&s_stop[0], static_cast<int>(threadIdx.x));     // the reverse scan runs from the last thread down
    __syncthreads();
    if (static_cast<int>(threadIdx.x) < s_stop[0]) { best_gain = kNegInf; best_thr = -1; any_valid = false; }
    for (int o = 16; o; o >>= 1) {
      const double og = __shfl_xor_sync(0xffffffffu, best_gain, o);
      const int ot = __shfl_xor_sync(0xffffffffu, best_thr, o);
      const double olg = __shfl_xor_sync(0xffffffffu, best_lg, o), olh = __shfl_xor_sync(0xffffffffu, best_lh, o);
      const int olc = __shfl_xor_sync(0xffffffffu, best_lc, o);
      if (og > best_gain || (og == best_gain && ot > best_thr)) { best_gain = og; best_thr = ot; best_lg = olg; best_lh = olh; best_lc = olc; }
    }
    if (lane == 0) { s_bg[warp] = best_gain; s_bt[warp] = best_thr; s_blg[warp] = best_lg; s_blh[warp] = best_lh; s_blc[warp] = best_lc; }
    __syncthreads();
    for (int w2 = 0; w2 < 8; ++w2)
      if (s_bg[w2] > best_gain || (s_bg[w2] == best_gain && s_bt[w2] > best_thr)) { best_gain = s_bg[w2]; best_thr = s_bt[w2]; best_lg = s_blg[w2]; best_lh = s_blh[w2]; best_lc = s_blc[w2]; }
    __syncthreads();
  }
  // ---- forward pass (NaN-as-missing features only): bins 0 .. num_bin-2, threshold = b, NaN goes right
  if (two_way) {
    const int hi = m.num_bin - 2;
    long long ag = 0, ah = 0, ac = 0, lg = 0, lh = 0, lc = 0;
    for (int b = b0; b < b1; ++b) {
      const long long qg = hist[b * 2], qh = hist[b * 2 + 1];
      const int c = static_cast<int>(static_cast<double>(qh) * inv_h * cnt_factor + 0.5);
      if (b >= 1 && b < m.num_bin) { ag += qg; ah += qh; ac += c; }
      if (b >= m.offset && b <= hi) { lg += qg; lh += qh; lc += c; }
    }
    {   // block totals of (ag, ah, ac)
      long long ta = ag, tb = ah, tc = ac;
      for (int o = 16; o; o >>= 1) { ta += __shfl_xor_sync(0xffffffffu, ta, o); tb += __shfl_xor_sync(0xffffffffu, tb, o); tc += __shfl_xor_sync(0xffffffffu, tc, o); }
      if (lane == 0) { s_sc[warp] = ta; s_sc[8 + warp] = tb; s_sc[16 + warp] = tc; }
      __syncthreads();
      if (threadIdx.x == 0) { long long x = 0, y = 0, z = 0; for (int w2 = 0; w2 < 8; ++w2) { x += s_sc[w2]; y += s_sc[8 + w2]; z += s_sc[16 + w2]; } s_tot[0] = x; s_tot[1] = y; s_tot[2] = z; }
      __syncthreads();
      ag = s_tot[0]; ah = s_tot[1]; ac = s_tot[2];
    }
    long long pg = lg, ph = lh, pc = lc;
    d_block_excl3(pg, ph, pc, 0, s_sc);
    double base_g = 0.0, base_h = kEpsD; int base_c = 0;
    if (m.offset == 1) {   // implicit bin 0 = leaf total - everything stored  [UPSTREAM NA_AS_MISSING && offset==1]
      base_g = sum_g - static_cast<double>(ag) * inv_g;
      base_h = (sum_h - kEpsD) - static_cast<double>(ah) * inv_h;
      base_c = num_data - static_cast<int>(ac);
    }
    double f_gain = kNegInf, f_lg = 0, f_lh = 0; int f_thr = 1 << 30, f_lc = 0;
    bool f_stop = false, f_valid = false;
    for (int b = b0; b < b1; ++b) {
      if (b > hi) continue;
      if (b >= m.offset) { const long long qh = hist[b * 2 + 1]; pg += hist[b * 2]; ph += qh; pc += static_cast<int>(static_cast<double>(qh) * inv_h * cnt_factor + 0.5); }
      const double slg = base_g + static_cast<double>(pg) * inv_g;
      const double slh = base_h + static_cast<double>(ph) * inv_h;
      const int left_count = base_c + static_cast<int>(pc);
      if (left_count < p.min_data_in_leaf || slh < p.min_sum_hessian) continue;
      const int right_count = num_data - left_count;
      const double srh = sum_h - slh;
      if (right_count < p.min_data_in_leaf || srh < p.min_sum_hessian) { f_stop = true; break; }
      if (kExtra && b != rand_thr) continue;
      const double srg = sum_g - slg;
      const double gain = kMono ? d_mono_split_gain(slg, slh, srg, srh, left_count, right_count, L.output, p, L.mono_min, L.mono_max, mono)
                                : d_leaf_gain(slg, slh, p) + d_leaf_gain(srg, srh, p);
      if (gain <= min_gain_shift) continue;
      f_valid = true;
      if (gain > f_gain) { f_gain = gain; f_lg = slg; f_lh = slh; f_thr = b; f_lc = left_count; }
    }
    if (f_stop) atomicMin(&s_stop[1], static_cast<int>(threadIdx.x));    // the forward scan runs from thread 0 up
    __syncthreads();
    if (static_cast<int>(threadIdx.x) > s_stop[1]) { f_gain = kNegInf; f_thr = 1 << 30; f_valid = false; }
    any_valid |= f_valid;
    for (int o = 16; o; o >>= 1) {
      const double og = __shfl_xor_sync(0xffffffffu, f_gain, o);
      const int ot = __shfl_xor_sync(0xffffffffu, f_thr, o);
      const double olg = __shfl_xor_sync(0xffffffffu, f_lg, o), olh = __shfl_xor_sync(0xffffffffu, f_lh, o);
      const int olc = __shfl_xor_sync(0xffffffffu, f_lc, o);
      if (og > f_gain || (og == f_gain && ot < f_thr)) { f_gain = og; f_thr = ot; f_lg = olg; f_lh = olh; f_lc = olc; }
    }
    if (lane == 0) { s_bg[warp] = f_gain; s_bt[warp] = f_thr; s_blg[warp] = f_lg; s_blh[warp] = f_lh; s_blc[warp] = f_lc; }
    __syncthreads();
    for (int w2 = 0; w2 < 8; ++w2)
      if (s_bg[w2] > f_gain || (s_bg[w2] == f_gain && s_bt[w2] < f_thr)) { f_gain = s_bg[w2]; f_thr = s_bt[w2]; f_lg = s_blg[w2]; f_lh = s_blh[w2]; f_lc = s_blc[w2]; }
    __syncthreads();
    if (f_gain > best_gain) { best_gain = f_gain; best_thr = f_thr; best_lg = f_lg; best_lh = f_lh; best_lc = f_lc; best_dl = 0; }
  } else if (m.missing_type == 2) {
    best_dl = 0;
  }
  if (any_valid) atomicOr(&s_any, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    SplitCand& out = *outp;
    *flag = s_any ? 1 : 0;
    out.is_cat = 0; out.default_left = 1;
    if (s_any && best_gain > min_gain_shift) {
      out.gain = best_gain - min_gain_shift; out.left_g = best_lg; out.left_h = best_lh; out.threshold = best_thr;
      out.left_count = best_lc; out.default_left = best_dl;
    }
  }
}

// ---- steps shared by the split scans k_scan and k_scan_wide (one block per (smaller|larger leaf, feature))
// the candidate of a feature that is not scanned, or before its scan found a split
__device__ __forceinline__ SplitCand d_empty_cand(int u) {
  SplitCand out;
  out.gain = kNegInf; out.left_g = 0; out.left_h = 0; out.threshold = 0; out.left_count = 0; out.default_left = 1; out.feature = u;
  out.l2_extra = 0; out.is_cat = 0; out.cat_list_len = 0;
  for (int wd = 0; wd < 8; ++wd) out.cat_bits[wd] = 0u;
  return out;
}
// ---- forced splits ([UPSTREAM] FeatureHistogram::GatherInfoForThreshold{Numerical,Categorical}): plan node nd on the leaf's reduced
// histogram column `hist` of its feature m, by every thread of the scan block of (leaf, feature); thread 0 stores the result in *outp.
// - numerical: the right side sums the bins above nd.bin, the NaN bin left out; the left side is the leaf total minus it, so NaN goes
//   left (default_left = 1).  Counts are rounded per bin from the hessians, as in the scans.
// - categorical: the left side is the single bin nd.bin, which must be one of the feature's category bins (not 0).
// The gain and min_gain_shift are the scans' (kMono: smoothed toward the leaf's output); the node is valid only when the gain exceeds
// min_gain_shift, and min_data_in_leaf and min_sum_hessian_in_leaf do not apply.  An invalid node stores gain -inf.  Out of line, with
// barriers before and after: the scan of the same block may overwrite `hist` when it is the block's scratch (a bundle member).
template <bool kMono>
__device__ __noinline__ void d_forced_eval(const long long* __restrict__ hist, const FeatMeta m, const ForcedNode nd, int u, int wide,
                                           const LeafState& L, double inv_g, double inv_h, const SplitParams& p, SplitCand* outp) {
  __shared__ long long s_fr[3][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double sum_g = L.sum_g, sum_h = L.sum_h + 2 * kEpsD;
  const int num_data = L.global_count;
  const double cnt_factor = num_data / sum_h;
  long long r[3] = {0, 0, 0};
  if (!nd.is_cat) {
    const int hi = m.num_bin - 1 - (m.missing_type == 2 ? 1 : 0);
    for (int b = nd.bin + 1 + static_cast<int>(threadIdx.x); b <= hi; b += blockDim.x) {
      const long long qh = hist[b * 2 + 1];
      r[0] += hist[b * 2]; r[1] += qh; r[2] += static_cast<int>(static_cast<double>(qh) * inv_h * cnt_factor + 0.5);
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
    for (int o = 16; o; o >>= 1) r[i] += __shfl_xor_sync(0xffffffffu, r[i], o);
  __syncthreads();
  if (lane == 0) for (int i = 0; i < 3; ++i) s_fr[i][warp] = r[i];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) { r[i] = 0; for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) r[i] += s_fr[i][w]; }
    bool ok = true;
    double lg, lh, rg, rh;
    int lc, rc;
    if (!nd.is_cat) {
      rg = static_cast<double>(r[0]) * inv_g; rh = kEpsD + static_cast<double>(r[1]) * inv_h; rc = static_cast<int>(r[2]);
      lc = num_data - rc; lg = sum_g - rg; lh = sum_h - rh;
    } else {
      ok = nd.bin > 0 && nd.bin < m.num_bin;
      const double g = ok ? static_cast<double>(hist[nd.bin * 2]) * inv_g : 0.0, h = ok ? static_cast<double>(hist[nd.bin * 2 + 1]) * inv_h : 0.0;
      lc = static_cast<int>(h * cnt_factor + 0.5); rc = num_data - lc;
      lg = g; lh = h + kEpsD; rg = sum_g - g; rh = sum_h - lh;
    }
    const double min_gain_shift = (kMono ? d_smooth_leaf_gain(sum_g, sum_h, num_data, L.output, p) : d_leaf_gain(sum_g, sum_h, p)) + p.min_gain_to_split;
    const double gain = kMono ? d_mono_split_gain(lg, lh, rg, rh, lc, rc, L.output, p, L.mono_min, L.mono_max, 0)
                              : d_leaf_gain(lg, lh, p) + d_leaf_gain(rg, rh, p);
    SplitCand out = d_empty_cand(u);
    if (ok && gain > min_gain_shift) {
      out.gain = gain - min_gain_shift; out.left_g = lg; out.left_h = lh; out.left_count = lc;
      out.threshold = nd.is_cat ? 0 : nd.bin; out.default_left = nd.is_cat ? 0 : 1; out.is_cat = nd.is_cat;
      if (nd.is_cat && wide) { out.cat_list_len = 1; out.cat_list[0] = static_cast<unsigned short>(nd.bin); }
      else if (nd.is_cat) out.cat_bits[nd.bin >> 5] = 1u << (nd.bin & 31);
    }
    *outp = out;
    __threadfence();      // before the block takes the kernel's scan ticket: the pick step reads it
  }
  __syncthreads();
}
// the plan node the scan block of `leaf` evaluates in this round, or -1: while the phase lasts, the round after node j - 1 was applied
// scans that node's two new leaves, and each of its child nodes is evaluated on its own leaf (the root's node 0 on leaf 0 in round 0)
__device__ __forceinline__ int d_forced_node(const TreeCtrl* ctrl, const ForcedArgs& f, int leaf) {
  const int j = ctrl->forced_next;
  if (j < 0) return -1;
  if (j == 0) return leaf == 0 ? 0 : -1;
  const ForcedNode& par = f.nodes[j - 1];
  if (par.left >= 0 && f.nodes[par.left].leaf == leaf) return par.left;
  if (par.right >= 0 && f.nodes[par.right].leaf == leaf) return par.right;
  return -1;
}
// the forced-split step of a scan block of (leaf, feature u) whose column `hist` holds the leaf's histogram: evaluates the plan node of
// this leaf and round if it splits on u.  Called by every thread; the condition is the same in all of them.
template <bool kMono>
__device__ __forceinline__ void d_forced_step(const TreeCtrl* ctrl, const ForcedArgs& f, int leaf, int u, const long long* hist, const FeatMeta& m,
                                              const LeafState& L, const SplitParams& p) {
  const int k = d_forced_node(ctrl, f, leaf);
  if (k >= 0 && f.nodes[k].feature == u)
    d_forced_eval<kMono>(hist, m, f.nodes[k], u, u >= p.nfn, L, ctrl->inv_g, ctrl->inv_h, p, &f.evals[k]);
}

// one thread: the candidate of (leaf `which`, feature u) and, for extra_trees, the scan's number of draws (see d_lcg_next), then a fence
// that makes both visible to the block that runs the pick step
template <bool kExtra>
__device__ __forceinline__ void d_publish_cand(SplitCand* cands, unsigned* xrand, const SplitParams& p, int which, int u, const SplitCand& out,
                                               int drew) {
  cands[which * p.nf_pad + u] = out;
  if (kExtra) xrand[static_cast<size_t>(1 + which) * p.nf_pad + u] = static_cast<unsigned>(drew);
  __threadfence();
}
// a feature's histogram column of n (g,h) pairs reduced into the leaf's pool slot: the smaller leaf's (which = 0) is H's, the larger's is
// parent - H (exact int64).  Ends with a barrier: the scan reads pairs other threads of the block reduced.
__device__ __forceinline__ void d_reduce_column(const long long* __restrict__ src, long long* __restrict__ dst, int n, int which) {
  for (int b = threadIdx.x; b < n; b += blockDim.x) {
    longlong2 sv = *reinterpret_cast<const longlong2*>(src + b * 2);
    if (which) { const longlong2 pr = *reinterpret_cast<const longlong2*>(dst + b * 2); sv.x = pr.x - sv.x; sv.y = pr.y - sv.y; }
    *reinterpret_cast<longlong2*>(dst + b * 2) = sv;
  }
  __syncthreads();
}
// a numerical feature u scanned by this block: extra_trees' draw from the feature's stream state xr (for the larger leaf already past the
// smaller leaf's draw, d_smaller_drew), the two-pass scan of its reduced histogram, and a monotone feature's candidate gain times
// d_mono_penalty at the leaf's depth.  Returns the number of draws taken.
template <bool kExtra, bool kMono>
__device__ __forceinline__ int d_scan_numeric_feature(const long long* __restrict__ hist, const FeatMeta& m, int u, const LeafState& L, double inv_g,
                                                      double inv_h, const SplitParams& p, uint8_t* flag, SplitCand* out, unsigned xr,
                                                      const ConstraintArgs& cons) {
  const int rand_thr = kExtra ? d_extra_draw(&xr, m.num_bin - 2) : 0;
  const int mono = kMono ? cons.type[u] : 0;
  d_scan_numeric<kExtra, kMono>(hist, m, L, inv_g, inv_h, p, flag, out, rand_thr, mono);
  if (kMono && mono != 0 && threadIdx.x == 0) out->gain *= d_mono_penalty(L.depth, cons.penalty);
  return m.num_bin > 2 ? 1 : 0;
}

// order of the wide categorical selection: side 0 ascending (key, bin), side 1 descending
__device__ __forceinline__ bool d_sel_prec(int side, double k, int b, double rk, int rb) {
  return side == 0 ? (k < rk || (k == rk && b < rb)) : (k > rk || (k == rk && b > rb));
}
constexpr int kSelList = 512;
// bitonic sort by 256 threads of TWO (key, id) arrays of n (power of two <= stride) entries: array 0 ascending, array 1 descending in
// (key, id); ends with a barrier
__device__ __noinline__ void d_block_bitonic2(double* k, int* id, int stride, int n) {
  for (int k2 = 2; k2 <= n; k2 <<= 1)
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int x = i ^ j;
        if (x <= i) continue;
        const bool up = (i & k2) == 0;
#pragma unroll
        for (int side = 0; side < 2; ++side) {
          double* kk = k + side * stride; int* ii = id + side * stride;
          const double ka = kk[i], kb = kk[x];
          const int ia = ii[i], ib = ii[x];
          const bool sw = up ? d_sel_prec(side, kb, ib, ka, ia) : d_sel_prec(side, ka, ia, kb, ib);
          if (sw) { kk[i] = kb; kk[x] = ka; ii[i] = ib; ii[x] = ia; }
        }
      }
    }
  __syncthreads();
}

// Split search of a WIDE categorical feature (FeatureHistogram::FindBestThresholdCategoricalInner, many-vs-many branch): one block per
// (smaller|larger, feature).  The histogram is reduced into the leaf's pool slot (parent - smaller for the larger child), the
// max_cat_threshold smallest and largest ctr = g / (h + cat_smooth) among the bins that hold >= cat_smooth rows are selected in the
// (ctr, bin) order of the reference's stable sort, and thread 0 accumulates from both ends exactly like the sequential code.
// kMono (monotone constraints or path smoothing): output-based gains and min_gain_shift as in d_scan_numeric / d_scan_feature_cat, and
// a monotone numerical feature's candidate gain times d_mono_penalty at the leaf's depth.
template <bool kExtra, bool kMono>
__global__ void __launch_bounds__(256)
k_scan_wide(const TreeCtrl* __restrict__ ctrl, const LeafState* __restrict__ leaves, const FeatMeta* __restrict__ meta, const long long* __restrict__ H,
            long long* __restrict__ pool, size_t slot_elems, uint8_t* __restrict__ flags, SplitCand* __restrict__ cands, SplitParams p,
            unsigned* __restrict__ xrand, ConstraintArgs cons, ForcedArgs forced) {
  extern __shared__ __align__(16) unsigned char sw_smem[];
  double* s_key = reinterpret_cast<double*>(sw_smem);                          // [num_bin] ctr keys of the used bins, +inf otherwise
  __shared__ int s_used;
  const int which = blockIdx.y, u = p.nfn + blockIdx.x;
  const int leaf = which ? ctrl->larger : ctrl->smaller;
  if (!ctrl->go || leaf < 0) return;
  SplitCand out = d_empty_cand(u);
  uint8_t* flag = &flags[static_cast<size_t>(leaf) * p.nf_pad + u];
  const FeatMeta m = meta[u];
  const LeafState& L = leaves[leaf];
  long long* dst = pool + static_cast<size_t>(L.hist_slot) * slot_elems + static_cast<size_t>(m.hist_off) * 2;
  const long long* src = H + static_cast<size_t>(m.hist_off) * 2;
  // forced splits: while the phase lasts every column of the scanned leaves is reduced, flagged or not, so that a plan node can be
  // evaluated on any used feature (its leaf's ancestors were all scanned in the phase)
  const bool forcing = forced.nodes && ctrl->forced_next >= 0;
  if (!*flag) {
    if (forcing) {
      d_reduce_column(src, dst, m.num_bin, which);
      d_forced_step<kMono>(ctrl, forced, leaf, u, dst, m, L, p);
    }
    if (threadIdx.x == 0) d_publish_cand<kExtra>(cands, xrand, p, which, u, out, 0);
    return;
  }
  const double inv_g = ctrl->inv_g, inv_h = ctrl->inv_h;
  const double sum_g = L.sum_g, sum_h = L.sum_h + 2 * kEpsD;
  const int num_data = L.global_count;
  const double cnt_factor = num_data / sum_h;
  // extra_trees: the stream state before this scan's draw (see d_smaller_drew); every categorical feature here is many-vs-many
  unsigned xr = kExtra ? xrand[u] : 0u;
  if (kExtra && which && d_smaller_drew(src, m, ctrl, leaves, p, min(p.max_cat_threshold, kCatListMax))) xr = d_lcg_next(xr);
  if (!m.is_categorical) {        // wide numerical feature (max_bin > 255): reduce into the pool slot, then the block-wide two-pass scan
    d_reduce_column(src, dst, m.num_bin, which);
    if (forcing) d_forced_step<kMono>(ctrl, forced, leaf, u, dst, m, L, p);
    const int drew = d_scan_numeric_feature<kExtra, kMono>(dst, m, u, L, inv_g, inv_h, p, flag, &out, xr, cons);
    if (threadIdx.x == 0) d_publish_cand<kExtra>(cands, xrand, p, which, u, out, drew);
    return;
  }
  // ---- reduce into the pool slot and build the ctr keys (loads of 4 bins in flight per thread before the dependent stores)
  if (threadIdx.x == 0) s_used = 0;
  __syncthreads();
  int my_used = 0;
  const double kPosInf = __longlong_as_double(0x7ff0000000000000LL);      // unused bins: never selected
  for (int b0 = threadIdx.x; b0 < m.num_bin; b0 += 4 * blockDim.x) {
    longlong2 sv[4], pr[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int b = b0 + q * blockDim.x;
      if (b < m.num_bin) {
        sv[q] = *reinterpret_cast<const longlong2*>(src + b * 2);
        if (which) pr[q] = *reinterpret_cast<const longlong2*>(dst + b * 2);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int b = b0 + q * blockDim.x;
      if (b >= m.num_bin) continue;
      longlong2 v = sv[q];
      if (which) { v.x = pr[q].x - v.x; v.y = pr[q].y - v.y; }
      *reinterpret_cast<longlong2*>(dst + b * 2) = v;
      const double g = static_cast<double>(v.x) * inv_g, h = static_cast<double>(v.y) * inv_h;
      const int cnt = static_cast<int>(h * cnt_factor + 0.5);
      double key = kPosInf;
      if (b >= 1 && cnt >= p.cat_smooth) { key = g / (h + p.cat_smooth); ++my_used; }
      s_key[b] = key;
    }
  }
  if (my_used) atomicAdd(&s_used, my_used);
  __syncthreads();
  if (forcing) d_forced_step<kMono>(ctrl, forced, leaf, u, dst, m, L, p);
  const int used_bin = s_used;
  const int max_num_cat = min(min(p.max_cat_threshold, kCatListMax), (used_bin + 1) / 2);
  int rand_i = 0, drew = 0;      // extra_trees: the one prefix length - 1 evaluated
  if (kExtra) {
    const int range = d_cat_rand_range(used_bin, min(p.max_cat_threshold, kCatListMax));
    rand_i = d_extra_draw(&xr, range);
    drew = range > 0 ? 1 : 0;
  }
  // ---- the reference sorts the used bins by (ctr, bin) and walks max_num_cat bins from either end; only those 2 * max_num_cat order
  // statistics are needed.  Sorting thousands of keys (first version: block-wide bitonic sort, ~600 us per launch) and selecting them
  // one per round (second version: 64 dependent rounds of a strided rescan, ~300 us — the rescan's latency is the same whether one
  // thread or all of them run it) both serialise on one SM.  Instead: (A) every thread takes the min and max of its own bins,
  // (B) the 256 per-thread minima (maxima) are sorted and the max_num_cat-th of them is a threshold that at least max_num_cat keys
  // reach, (C) the keys within the threshold are appended to a short list (typically max_num_cat + a few), (D) the list is sorted.
  // Three passes over the keys instead of 2 * max_num_cat.  The (key, bin) order is total, so the result equals the stable sort.
  __shared__ unsigned short s_sel[2][kCatListMax];
  __shared__ double s_selg[2][kCatListMax], s_selh[2][kCatListMax];
  __shared__ double s_rk[8];
  __shared__ int s_ri[8];
  __shared__ double s_tk[2][256], s_lk[2][kSelList];
  __shared__ int s_ti[2][256], s_li[2][kSelList];
  __shared__ int s_cnt[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  bool overflow = false;
  if (max_num_cat > 0) {
    double ak = kPosInf, zk = kNegInf; int ai = 0x7fffffff, zi = -1;
    for (int b = threadIdx.x; b < m.num_bin; b += blockDim.x) {
      const double k = s_key[b];
      if (!(k < kPosInf)) continue;
      if (k < ak) { ak = k; ai = b; }
      if (k >= zk) { zk = k; zi = b; }
    }
    s_tk[0][threadIdx.x] = ak; s_ti[0][threadIdx.x] = ai; s_tk[1][threadIdx.x] = zk; s_ti[1][threadIdx.x] = zi;
    if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
    d_block_bitonic2(&s_tk[0][0], &s_ti[0][0], 256, 256);
    const double t0k = s_tk[0][max_num_cat - 1], t1k = s_tk[1][max_num_cat - 1];
    const int t0i = s_ti[0][max_num_cat - 1], t1i = s_ti[1][max_num_cat - 1];
    for (int b = threadIdx.x; b < m.num_bin; b += blockDim.x) {
      const double k = s_key[b];
      if (!(k < kPosInf)) continue;
      if (!d_sel_prec(0, t0k, t0i, k, b)) { const int pos = atomicAdd(&s_cnt[0], 1); if (pos < kSelList) { s_lk[0][pos] = k; s_li[0][pos] = b; } }
      if (!d_sel_prec(1, t1k, t1i, k, b)) { const int pos = atomicAdd(&s_cnt[1], 1); if (pos < kSelList) { s_lk[1][pos] = k; s_li[1][pos] = b; } }
    }
    __syncthreads();
    const int n0 = s_cnt[0], n1 = s_cnt[1];
    overflow = n0 > kSelList || n1 > kSelList;      // e.g. all small keys on bins congruent mod 256: fall back to the round-based selection
    if (!overflow) {
      int n2 = 2;
      while (n2 < n0 || n2 < n1) n2 <<= 1;
      for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        if (i >= n0) { s_lk[0][i] = kPosInf; s_li[0][i] = 0x7fffffff; }
        if (i >= n1) { s_lk[1][i] = kNegInf; s_li[1][i] = -1; }
      }
      d_block_bitonic2(&s_lk[0][0], &s_li[0][0], kSelList, n2);
      if (threadIdx.x < 2 * max_num_cat) {
        const int side = threadIdx.x / max_num_cat, i = threadIdx.x - side * max_num_cat;
        s_sel[side][i] = static_cast<unsigned short>(s_li[side][i]);
      }
    }
  }
  // fallback (list overflow): tournament — every thread keeps the best remaining key of ITS bins (b = tid + 256 j); a round reduces the
  // 256 cached candidates and only the winner's owner rescans its own bins
  if (overflow)
  for (int side = 0; side < 2; ++side) {
    auto better = [&](double k, int b, double rk, int rb) -> bool {      // (k, b) precedes (rk, rb) on this side; rb sentinel = nothing yet
      if (side == 0) return rb == 0x7fffffff || k < rk || (k == rk && b < rb);
      return rb == -1 || k > rk || (k == rk && b > rb);
    };
    auto own_next = [&](double pk, int pi, double* ok, int* oi) {         // best own key strictly beyond (pk, pi)
      double bk = 0.0; int bi = side == 0 ? 0x7fffffff : -1;
      for (int b = threadIdx.x; b < m.num_bin; b += blockDim.x) {
        const double k = s_key[b];
        if (!(k < kPosInf)) continue;
        const bool beyond = side == 0 ? (k > pk || (k == pk && b > pi)) : (k < pk || (k == pk && b < pi));
        if (beyond && better(k, b, bk, bi)) { bk = k; bi = b; }
      }
      *ok = bk; *oi = bi;
    };
    const int none = side == 0 ? 0x7fffffff : -1;
    double ck; int ci;
    own_next(side == 0 ? kNegInf : kPosInf, side == 0 ? -1 : 0x7fffffff, &ck, &ci);
    for (int r = 0; r < max_num_cat; ++r) {
      double bk = ck; int bi = ci;
      for (int o = 16; o; o >>= 1) {
        const double ok = __shfl_xor_sync(0xffffffffu, bk, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi != none && better(ok, oi, bk, bi)) { bk = ok; bi = oi; }
      }
      if (lane == 0) { s_rk[warp] = bk; s_ri[warp] = bi; }
      __syncthreads();
      bk = s_rk[0]; bi = s_ri[0];
      for (int w2 = 1; w2 < 8; ++w2) if (s_ri[w2] != none && better(s_rk[w2], s_ri[w2], bk, bi)) { bk = s_rk[w2]; bi = s_ri[w2]; }
      __syncthreads();
      if (threadIdx.x == 0) s_sel[side][r] = static_cast<unsigned short>(bi);      // exists: r < max_num_cat <= used_bin
      if (bi != none && (bi & 255) == static_cast<int>(threadIdx.x)) own_next(bk, bi, &ck, &ci);      // only the owner of the winner moves on
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 * max_num_cat) {
    const int side = threadIdx.x / max_num_cat, i = threadIdx.x - side * max_num_cat;
    const int t = s_sel[side][i];
    s_selg[side][i] = static_cast<double>(dst[t * 2]) * inv_g;
    s_selh[side][i] = static_cast<double>(dst[t * 2 + 1]) * inv_h;
  }
  __syncthreads();
  // the walk from either end is sequential only in its cheap state (running sums, the min_data_per_group counter, continue / break); lane 0
  // of warps 0 and 1 run it for one direction each and mark the prefixes the reference evaluates, the gains (fp64 divisions) are then
  // computed one prefix per thread, and thread 0 takes the first maximum in the reference's (direction, i) order
  __shared__ double s_plg[2][kCatListMax], s_plh[2][kCatListMax], s_pgain[2][kCatListMax];
  __shared__ int s_plc[2][kCatListMax];
  if (threadIdx.x < 2 * kCatListMax) s_pgain[threadIdx.x / kCatListMax][threadIdx.x % kCatListMax] = kNegInf;
  __syncthreads();
  if (lane == 0 && warp < 2) {
    const int d = warp;
    int i = 0;
    d_cat_walk<kExtra>(used_bin, max_num_cat, num_data, sum_h, cnt_factor, p, rand_i,
                       [&](double* g, double* h) { *g = s_selg[d][i]; *h = s_selh[d][i]; ++i; },
                       [&](int j, double slg, double slh, double, int left_count) {
                         s_plg[d][j] = slg; s_plh[d][j] = slh; s_plc[d][j] = left_count; s_pgain[d][j] = 0.0;      // 0.0 = "evaluate me"
                       });
  }
  __syncthreads();
  const double min_gain_shift = (kMono ? d_smooth_leaf_gain(sum_g, sum_h, num_data, L.output, p) : d_leaf_gain(sum_g, sum_h, p)) + p.min_gain_to_split;
  if (threadIdx.x < 2 * kCatListMax) {
    const int d = threadIdx.x / kCatListMax, i = threadIdx.x % kCatListMax;
    if (s_pgain[d][i] == 0.0) {
      SplitParams pc = p;
      pc.l2 += p.cat_l2;
      const double slg = s_plg[d][i], slh = s_plh[d][i];
      s_pgain[d][i] = kMono ? d_mono_split_gain(slg, slh, sum_g - slg, sum_h - slh, s_plc[d][i], num_data - s_plc[d][i], L.output, pc,
                                                L.mono_min, L.mono_max, 0)
                            : d_leaf_gain(slg, slh, pc) + d_leaf_gain(sum_g - slg, sum_h - slh, pc);
    }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  bool any_valid = false;
  double best_gain = kNegInf, best_lg = 0, best_lh = 0;
  int best_i = -1, best_dir = 1, best_lc = 0;
  for (int d = 0; d < 2; ++d)
    for (int i = 0; i < max_num_cat; ++i) {
      const double gain = s_pgain[d][i];
      if (!(gain > min_gain_shift)) continue;      // also skips the -inf of the prefixes the walk did not evaluate
      any_valid = true;
      if (gain > best_gain) { best_gain = gain; best_lg = s_plg[d][i]; best_lh = s_plh[d][i]; best_lc = s_plc[d][i]; best_i = i; best_dir = d == 0 ? 1 : -1; }
    }
  *flag = any_valid ? 1 : 0;
  if (any_valid) {
    out.gain = best_gain - min_gain_shift; out.left_g = best_lg; out.left_h = best_lh; out.threshold = 0; out.left_count = best_lc;
    out.default_left = 0; out.is_cat = 1; out.l2_extra = p.cat_l2;
    out.cat_list_len = best_i + 1;
    for (int i = 0; i <= best_i && i < kCatListMax; ++i) out.cat_list[i] = s_sel[best_dir == 1 ? 0 : 1][i];
  }
  d_publish_cand<kExtra>(cands, xrand, p, which, u, out, drew);
}

// A bundle member's histogram out of its bundle column, by the member's k_scan block (thread t = column slot t).  The member's slots of
// the column become its bins != mfb; this block alone updates them in the pool (smaller leaf: H, larger: parent - H).  Every column of a leaf
// sums to the leaf total, so the smaller leaf's total is this column of H summed, and the larger's is its parent's total minus that; the
// member's mfb is the total minus its other bins.  All exact int64, so `out` equals the unbundled feature's histogram bit for bit.
// tot != null (the voting learner's global scan): src is the leaf's reduced column and tot its reduced (g,h) total; dst and L are untouched.
// leaf_tot != null: the leaf total used is also stored there (shared memory, read by the block after the call).
__device__ __noinline__ void d_unbundle_hist(const long long* __restrict__ src, long long* __restrict__ dst, int num_bin, int mfb, int base, int which,
                                             LeafState* L, longlong2* out, const long long* __restrict__ tot = nullptr,
                                             longlong2* leaf_tot = nullptr) {
  __shared__ long long s_red[4][8];
  const int b = threadIdx.x, lane = b & 31, warp = b >> 5;
  const longlong2 hv = reinterpret_cast<const longlong2*>(src)[b];
  const bool own = b > base && b < base + num_bin;
  longlong2 sv = hv;
  if (own) {
    if (which && !tot) { const longlong2 pr = reinterpret_cast<const longlong2*>(dst)[b]; sv.x = pr.x - hv.x; sv.y = pr.y - hv.y; }
    if (!tot) reinterpret_cast<longlong2*>(dst)[b] = sv;
    const int v = b - base - 1;
    out[v < mfb ? v : v + 1] = sv;
  }
  long long r[4] = {hv.x, hv.y, own ? sv.x : 0, own ? sv.y : 0};
#pragma unroll
  for (int i = 0; i < 4; ++i)
    for (int o = 16; o; o >>= 1) r[i] += __shfl_xor_sync(0xffffffffu, r[i], o);
  if (lane == 0) for (int i = 0; i < 4; ++i) s_red[i][warp] = r[i];
  __syncthreads();
  if (b == 0) {
    long long t[4] = {0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) for (int w = 0; w < 8; ++w) t[i] += s_red[i][w];
    long long tg, th;
    if (tot) { tg = tot[0]; th = tot[1]; }
    else {
      tg = which ? L->qpar[0] - t[0] : t[0]; th = which ? L->qpar[1] - t[1] : t[1];
      L->qtot[0] = tg; L->qtot[1] = th;      // every member block of this leaf writes the same value
    }
    out[mfb] = make_longlong2(tg - t[2], th - t[3]);
    if (leaf_tot) *leaf_tot = make_longlong2(tg, th);
  }
  __syncthreads();
}

// ---------------------------------------------------------------- K5/K6 for the tile features: one BLOCK per (smaller|larger, feature)
// Thread t = bin t.  The block reduces the feature into the leaf's pool slot (larger child: parent - smaller, exact int64), then runs the
// same block-wide two-pass scan as the wide numerical features (d_scan_numeric with one bin per thread: exclusive block scans of
// (g, h, count), one candidate per thread and direction, block argmax with the sequential tie-breaks) — the dependent chain of software
// fp64 divisions per thread is 2 long instead of 16 as in the round-1 warp-per-feature scan, and the code is shared and small (the old
// kernel was instruction-fetch bound).  Categorical tile features keep the warp-level search (d_scan_feature_cat) on warp 0.  The block that
// finishes last picks the best candidate per leaf and the next leaf to split.
//
// The voting-parallel learner ([UPSTREAM] VotingParallelTreeLearner) runs the same kernel twice per split, with kMode:
//   kScanLocal   every block writes its column of the LOCAL histograms into the pool whatever the feature's flag (the pool holds local
//                histograms; the larger child is local parent - local smaller), takes the leaf's exact local (g,h) total from its column
//                of H (every storage column of a leaf sums to the leaf's total: smaller = H's column, larger = parent total - that; kept in
//                LeafState::qtot / qpar), and scans flagged features with the local split parameters `p`, the local sums and the leaf's
//                true local row count.  This scan alone writes the is_splittable flags.  Its last block selects each leaf's local top-k
//                candidates into the vote records (d_topk_block) instead of picking.
//   kScanGlobal  a feature voted for the leaf (VoteBufs::voted) is scanned from its column of the reduced buffer (k_vote_pack) with the
//                global split parameters and leaf sums, whatever its local flag; every other feature yields a -inf candidate.  No flag
//                is written, and the last block runs the pick step as the data-parallel learner does.
constexpr int kScanPlain = 0, kScanLocal = 1, kScanGlobal = 2;
struct VoteRec { int feature, left_count, right_count, pad; double gain; };     // feature: inner index, -1 for no candidate
// packed (reduced) buffer: [0, 4) the (qg, qh) totals of the smaller and the larger leaf, then 2 * top_k storage columns of 256 (g,h) pairs:
// column which * top_k + k is the k-th voted feature of leaf `which` (0 smaller, 1 larger), zero when the vote has fewer features
constexpr int kVoteTotals = 4;
constexpr int kVoteColumn = 512;
constexpr int kVoteMaxRecords = 2048;      // records of one leaf over all ranks that k_vote_pack handles (8 per thread)
struct VoteBufs {
  VoteRec* recs;              // [2][top_k] this rank's local top-k records (kScanLocal writes them)
  const int* voted;           // [2][top_k] voted inner features, -1: none (k_vote_pack writes them)
  const long long* packed;    // reduced packed buffer
  int top_k;
};

// this block's leaf's exact (qg, qh) sums of a 256-pair column (thread t = pair t), on every thread
__device__ __forceinline__ longlong2 d_block_sum_column(const long long* __restrict__ col) {
  __shared__ long long s_red[2][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  longlong2 v = reinterpret_cast<const longlong2*>(col)[threadIdx.x];
  for (int o = 16; o; o >>= 1) { v.x += __shfl_xor_sync(0xffffffffu, v.x, o); v.y += __shfl_xor_sync(0xffffffffu, v.y, o); }
  if (lane == 0) { s_red[0][warp] = v.x; s_red[1][warp] = v.y; }
  __syncthreads();
  longlong2 t = make_longlong2(0, 0);
  for (int w = 0; w < 8; ++w) { t.x += s_red[0][w]; t.y += s_red[1][w]; }
  __syncthreads();
  return t;
}

// The local top-k of both leaves ([UPSTREAM] VotingParallelTreeLearner::FindBestSplits, ArrayArgs::MaxK on SplitInfo::operator>): round k
// takes the best candidate after round k-1's in the order (gain desc, real feature index asc), threads 0..127 for the smaller leaf and
// 128..255 for the larger as in d_pick_block.  A -inf candidate, or no leaf, gives a record with feature -1.
__device__ __noinline__ void
d_topk_block(const TreeCtrl* ctrl, const LeafState* leaves, const FeatMeta* __restrict__ meta, const SplitCand* cands, const SplitParams& p,
             VoteRec* recs, int top_k) {
  __shared__ double s_gain[8], s_prev_gain[2];
  __shared__ int s_feat[8], s_idx[8], s_prev_feat[2];
  const int which = threadIdx.x >> 7, t = threadIdx.x & 127, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int leaf = ctrl->go ? (which ? ctrl->larger : ctrl->smaller) : -1;
  double pg = __longlong_as_double(0x7ff0000000000000LL);      // +inf: every candidate comes after it
  int pf = -1;
  for (int k = 0; k < top_k; ++k) {
    double bg = kNegInf; int bf = 0x7fffffff, bi = -1;
    if (leaf >= 0) {
      for (int u = t; u < p.nf; u += 128) {
        const double cg = __ldcg(&cands[which * p.nf_pad + u].gain);
        const int rf = meta[u].real_index;
        if (!(cg < pg || (cg == pg && rf > pf))) continue;      // taken in an earlier round
        if (bi < 0 || cg > bg || (cg == bg && rf < bf)) { bg = cg; bf = rf; bi = u; }
      }
    }
    for (int o = 16; o; o >>= 1) {
      const double og = __shfl_xor_sync(0xffffffffu, bg, o);
      const int of = __shfl_xor_sync(0xffffffffu, bf, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || og > bg || (og == bg && of < bf))) { bg = og; bf = of; bi = oi; }
    }
    if (lane == 0) { s_gain[warp] = bg; s_feat[warp] = bf; s_idx[warp] = bi; }
    __syncthreads();
    if (t == 0) {
      for (int w = which * 4; w < which * 4 + 4; ++w)
        if (s_idx[w] >= 0 && (bi < 0 || s_gain[w] > bg || (s_gain[w] == bg && s_feat[w] < bf))) { bg = s_gain[w]; bf = s_feat[w]; bi = s_idx[w]; }
      VoteRec r{-1, 0, 0, 0, kNegInf};
      if (bi >= 0 && bg > kNegInf) {
        const int lc = __ldcg(&cands[which * p.nf_pad + bi].left_count);
        r.feature = bi; r.gain = bg; r.left_count = lc; r.right_count = leaves[leaf].count - lc;
      }
      recs[which * top_k + k] = r;
      s_prev_gain[which] = bi >= 0 ? bg : kNegInf; s_prev_feat[which] = bi >= 0 ? bf : 0x7fffffff;
    }
    __syncthreads();
    pg = s_prev_gain[which]; pf = s_prev_feat[which];
  }
}

// extra_trees, in the block that runs the pick step once every scan block of the round (k_scan_wide's before them) has finished: advance
// each feature's stream by the draws of the round's smaller and larger leaf.  Features that were not scanned wrote 0.
__device__ __noinline__ void d_extra_commit(const TreeCtrl* ctrl, unsigned* xrand, const SplitParams& p) {
  if (!ctrl->go) return;
  const bool larger = ctrl->larger >= 0;
  for (int u = threadIdx.x; u < p.nf; u += blockDim.x) {
    unsigned n = __ldcg(&xrand[p.nf_pad + u]) + (larger ? __ldcg(&xrand[2 * p.nf_pad + u]) : 0u);
    unsigned x = xrand[u];
    for (; n > 0; --n) x = d_lcg_next(x);
    xrand[u] = x;
  }
}

// ---------------------------------------------------------------- per-node feature sampling
// The LCG of Random (d_lcg_next) advanced d steps at once: x -> A x + C, composed from the one-step map by squaring.
__device__ __forceinline__ void d_lcg_jump_map(unsigned d, unsigned* A, unsigned* C) {
  unsigned a = 214013u, c = 2531011u, ra = 1u, rc = 0u;
  for (; d; d >>= 1) {
    if (d & 1u) { ra = a * ra; rc = a * rc + c; }
    c = a * c + c; a = a * a;
  }
  *A = ra; *C = rc;
}
__device__ __forceinline__ unsigned d_lcg_jump(unsigned x, unsigned d) { unsigned A, C; d_lcg_jump_map(d, &A, &C); return A * x + C; }
// Random::Sample(n, k) (bin_mapper.h LcgRandom::Sample): whether it takes the selection branch, and how many draws it takes
__device__ __forceinline__ bool d_sample_selects(int n, int k) { return k > 1 && k > (n / log2(static_cast<double>(k))); }
__device__ __forceinline__ unsigned d_sample_draws(int n, int k) { return (k <= 0 || k >= n) ? 0u : (d_sample_selects(n, k) ? n : k); }

// The node sample of the round's leaf `which` ([UPSTREAM] ColSampler::GetByNode with feature_fraction_bynode < 1), run by one extra
// block per leaf in the k_scan grid, alongside the scan blocks; the pick step in the kernel's last block reads the masks.
// - pool: the tree's feature_fraction sample in real-index order, filtered to the features the leaf's interaction mask allows; n = |pool|.
// - k = min(a.k, n), with a.k = GetCnt(|tree sample|, feature_fraction_bynode) from the host.
// - the sample is Random::Sample(n, k) on the ColSampler stream: the smaller leaf's from the round's state, the larger leaf's from that
//   state advanced by the smaller leaf's draws (which depend only on its (n, k)), so both blocks draw at once.  The larger leaf's block
//   (or the smaller's, when the round has one leaf) writes the state after the round to col_next; the pick step commits it.
// - selection branch (n draws): warp 0 makes 32 draws at a time, one per lane, from jumps of the stream.  Position i is taken iff
//   NextFloat() < (k - c) / (n - i), c = positions taken so far.  NextFloat() = m / 32768 with m < 2^15, and a rational a / b with
//   b < 2^31 that differs from m / 32768 differs by at least 2^-15 / b, more than half an ulp of m / 32768, so the fp64 quotient is
//   below m / 32768 exactly when a / b is: the test is c < k - floor(m (n - i) / 2^15), a threshold each lane computes on its own.
//   The lanes' thresholds then pass through the dependent chain c += (c < t) in registers, 32 steps per warp shuffle round.
// - Floyd's branch (k draws): step s draws v_s in [0, r_s), r_s = n - k + s, and takes v_s unless it is taken already, else r_s.  v_s is
//   taken before step s iff an earlier step drew the same value (first[v] = the earliest step that drew v), or v_s = r_s' of an earlier
//   step s' that took its r.  Every thread resolves its steps from those two facts, repeating while any step changes (the chains of
//   the second kind are short), so no step waits on the one before it.
__device__ __noinline__ void d_bynode_sample(TreeCtrl* ctrl, const LeafState* leaves, const SplitParams& p,
                                             const unsigned long long* __restrict__ sets_of, NodeSampleArgs a) {
  const int which = blockIdx.y;
  const int leaf = which ? ctrl->larger : ctrl->smaller;
  if (!ctrl->go || leaf < 0) return;
  __shared__ int s_warp[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* mask = a.mask + static_cast<size_t>(which) * p.nf_pad;
  int* pool = a.work + static_cast<size_t>(which) * 4 * p.nf_pad;
  int* first = pool + p.nf_pad;
  int* vs = first + p.nf_pad;
  int* col = vs + p.nf_pad;
  const unsigned long long im = p.interaction ? leaves[leaf].inter_mask : ~0ull;
  const unsigned long long sm = p.interaction ? leaves[ctrl->smaller].inter_mask : ~0ull;
  int n = 0, n_smaller = 0;
  for (int i0 = 0; i0 < p.nf; i0 += blockDim.x) {      // ordered compaction of the pool; the same trip count in every thread
    const int i = i0 + threadIdx.x;
    bool in = false, in_smaller = false;
    int u = 0;
    if (i < p.nf) {
      u = a.order[i];
      mask[u] = 0;
      const bool used = a.tree_used[u] != 0;
      in = used && (!p.interaction || (sets_of[u] & im));
      in_smaller = used && (!p.interaction || (sets_of[u] & sm));
    }
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) s_warp[warp] = __popc(bal);
    n_smaller += __syncthreads_count(in_smaller);
    int at = n + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) at += s_warp[w];
    if (in) pool[at] = u;
    n += __syncthreads_count(in);
  }
  const int k = min(a.k, n);
  unsigned x0 = ctrl->col_state;
  if (which) x0 = d_lcg_jump(x0, d_sample_draws(n_smaller, min(a.k, n_smaller)));
  if (threadIdx.x == 0 && (which || ctrl->larger < 0)) ctrl->col_next = d_lcg_jump(x0, d_sample_draws(n, k));
  if (k <= 0) {
  } else if (k == n) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) mask[pool[i]] = 1;
  } else if (d_sample_selects(n, k)) {
    if (warp == 0) {
      unsigned Aj, Cj, A32, C32;
      d_lcg_jump_map(lane + 1, &Aj, &Cj);
      d_lcg_jump_map(32, &A32, &C32);
      unsigned base = x0;
      int c = 0;
      for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const unsigned m = ((Aj * base + Cj) >> 16) & 0x7fffu;
        base = A32 * base + C32;
        const int t = i < n ? k - static_cast<int>((static_cast<unsigned long long>(m) * static_cast<unsigned>(n - i)) >> 15) : INT_MIN;
        const int u = i < n ? pool[i] : 0;
        unsigned taken = 0u;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int tj = __shfl_sync(0xffffffffu, t, j);
          const int s = c < tj ? 1 : 0;
          taken |= static_cast<unsigned>(s) << j;
          c += s;
        }
        if ((taken >> lane) & 1u) mask[u] = 1;
      }
    }
  } else {
    const int r0 = n - k;
    for (int i = threadIdx.x; i < n; i += blockDim.x) first[i] = INT_MAX;
    __syncthreads();
    unsigned A, C;
    d_lcg_jump_map(blockDim.x, &A, &C);
    unsigned x = d_lcg_jump(x0, threadIdx.x + 1);
    for (int s = threadIdx.x; s < k; s += blockDim.x) {
      const int v = static_cast<int>((x & 0x7fffffffu) % static_cast<unsigned>(r0 + s));
      vs[s] = v;
      atomicMin(&first[v], s);
      x = A * x + C;
    }
    __syncthreads();
    for (int s = threadIdx.x; s < k; s += blockDim.x) col[s] = first[vs[s]] < s ? 1 : 0;
    for (;;) {
      __syncthreads();
      int changed = 0;
      for (int s = threadIdx.x; s < k; s += blockDim.x) {
        const int v = vs[s];
        if (!col[s] && v >= r0 && *reinterpret_cast<volatile int*>(&col[v - r0])) { col[s] = 1; changed = 1; }
      }
      if (!__syncthreads_or(changed)) break;
    }
    for (int s = threadIdx.x; s < k; s += blockDim.x) mask[pool[col[s] ? r0 + s : vs[s]]] = 1;
  }
  __threadfence();      // every thread's mask bytes, before thread 0 takes the kernel's scan ticket
}

// kMono (monotone constraints or path smoothing): the output-based scans (d_scan_numeric, d_scan_feature_cat), a monotone feature's
// candidate gain times d_mono_penalty at the leaf's depth, and outputs smoothed and clamped to the leaf's bounds in the pick step.
// Without a constraint list the bounds stay (-inf, +inf) and every type is 0, so only the smoothing remains.
template <int kMode, bool kExtra = false, bool kMono = false>
__global__ void __launch_bounds__(256, 4)
k_scan(TreeCtrl* ctrl, LeafState* leaves, const FeatMeta* __restrict__ meta,
       const long long* __restrict__ H, long long* __restrict__ pool, size_t slot_elems, uint8_t* __restrict__ flags,
       SplitCand* cands, SplitParams p, const int* __restrict__ bundle_base, VoteBufs vote, unsigned* __restrict__ xrand, ConstraintArgs cons,
       NodeSampleArgs node, ForcedArgs forced) {
  // dynamic scratch (kScanSmem, only when the dataset has categorical tile features or a bundle): the categorical search's work space,
  // or a bundle member's histogram (d_unbundle_hist)
  extern __shared__ double scan_ws[];
  static_assert(!kExtra || kMode == kScanPlain, "the voting learner does not train extra trees (Booster fails at create)");
  static_assert(!kMono || kMode == kScanPlain, "the voting learner does not train monotone constraints (Booster fails at create)");
  const int which = blockIdx.y;
  const int leaf = which ? ctrl->larger : ctrl->smaller;
  const int u = blockIdx.x;
  if (ctrl->go && leaf >= 0 && u < p.nfn) {
    SplitCand out = d_empty_cand(u);
    int drew = 0;      // extra_trees: this scan's number of draws (0 when the feature is not scanned)
    if constexpr (kMode == kScanGlobal) {
      int col = -1;
      for (int k = 0; k < vote.top_k; ++k) if (vote.voted[which * vote.top_k + k] == u) col = which * vote.top_k + k;
      if (col >= 0) {
        __shared__ uint8_t s_no_flag;      // the global scan writes no is_splittable flag
        const LeafState& L = leaves[leaf];
        const FeatMeta fm = meta[u];
        const long long* hist = vote.packed + kVoteTotals + static_cast<size_t>(col) * kVoteColumn;
        if (bundle_base && bundle_base[u] >= 0) {
          d_unbundle_hist(hist, nullptr, fm.num_bin, fm.default_bin, bundle_base[u], which, nullptr, reinterpret_cast<longlong2*>(scan_ws),
                          vote.packed + 2 * which);
          hist = reinterpret_cast<const long long*>(scan_ws);
        }
        if (!fm.is_categorical) {
          d_scan_numeric<false, false>(hist, fm, L, ctrl->inv_g, ctrl->inv_h, p, &s_no_flag, &out, 0, 0);
        } else if (threadIdx.x < 32) {
          long long qg[8], qh[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) { const int b = threadIdx.x * 8 + j; qg[j] = hist[b * 2]; qh[j] = hist[b * 2 + 1]; }
          d_scan_feature_cat<false, false>(qg, qh, threadIdx.x, fm, L, ctrl->inv_g, ctrl->inv_h, p, &s_no_flag, &out, scan_ws, 0u);
        }
      }
    } else {
      uint8_t* flag = &flags[static_cast<size_t>(leaf) * p.nf_pad + u];
      // forced splits: while the phase lasts every column of the scanned leaves is reduced, as in k_scan_wide
      const bool forcing = kMode == kScanPlain && forced.nodes && ctrl->forced_next >= 0;
      if (kMode == kScanLocal || *flag || forcing) {
        const FeatMeta fm = meta[u];
        long long* dst = pool + static_cast<size_t>(leaves[leaf].hist_slot) * slot_elems + static_cast<size_t>(fm.hist_off) * 2;
        const long long* src = H + static_cast<size_t>(fm.hist_off) * 2;
        const bool bundled = bundle_base && bundle_base[u] >= 0;
        __shared__ longlong2 s_leaf_tot;      // kScanLocal, bundle member: the leaf's local total from d_unbundle_hist
        if (!bundled) {
          d_reduce_column(src, dst, 256, which);      // the whole storage column: k_vote_pack reads whole columns of the pool
        } else {
          d_unbundle_hist(src, dst, fm.num_bin, fm.default_bin, bundle_base[u], which, leaves + leaf, reinterpret_cast<longlong2*>(scan_ws),
                          nullptr, kMode == kScanLocal ? &s_leaf_tot : nullptr);
          dst = reinterpret_cast<long long*>(scan_ws);
        }
        LeafState Lloc;      // kScanLocal: the leaf's local sums and true local row count
        if constexpr (kMode == kScanLocal) {
          LeafState& Lw = leaves[leaf];
          longlong2 lt = s_leaf_tot;      // a bundle member's d_unbundle_hist also wrote it to qtot
          if (!bundled) {
            const longlong2 t = d_block_sum_column(src);
            lt = which ? make_longlong2(Lw.qpar[0] - t.x, Lw.qpar[1] - t.y) : t;
            if (threadIdx.x == 0) { Lw.qtot[0] = lt.x; Lw.qtot[1] = lt.y; }      // every block of this leaf writes the same value
          }
          Lloc.sum_g = static_cast<double>(lt.x) * ctrl->inv_g; Lloc.sum_h = static_cast<double>(lt.y) * ctrl->inv_h;
          Lloc.global_count = Lw.count;
        }
        const LeafState& L = kMode == kScanLocal ? Lloc : leaves[leaf];
        if (forcing) d_forced_step<kMono>(ctrl, forced, leaf, u, dst, fm, L, p);
        if (*flag) {
          // extra_trees: the stream state before this scan's draw (see d_smaller_drew)
          unsigned xr = kExtra ? xrand[u] : 0u;
          if (kExtra && which && d_smaller_drew(src, fm, ctrl, leaves, p, p.max_cat_threshold)) xr = d_lcg_next(xr);
          if (!fm.is_categorical) {
            drew = d_scan_numeric_feature<kExtra, kMono>(dst, fm, u, L, ctrl->inv_g, ctrl->inv_h, p, flag, &out, xr, cons);
          } else if (threadIdx.x < 32) {
            long long qg[8], qh[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { const int b = threadIdx.x * 8 + j; qg[j] = dst[b * 2]; qh[j] = dst[b * 2 + 1]; }
            drew = d_scan_feature_cat<kExtra, kMono>(qg, qh, threadIdx.x, fm, L, ctrl->inv_g, ctrl->inv_h, p, flag, &out, scan_ws, xr);
          }
        }
      }
    }
    if (threadIdx.x == 0) d_publish_cand<kExtra>(cands, xrand, p, which, u, out, drew);
  } else if constexpr (kMode == kScanPlain) {
    if (node.mask && u == static_cast<int>(gridDim.x) - 1) d_bynode_sample(ctrl, leaves, p, cons.sets_of, node);      // the grid's extra column
  }
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned t = atomicAdd(&ctrl->scan_ticket, 1u);
    s_last = (t == gridDim.x * gridDim.y - 1) ? 1 : 0;
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    if constexpr (kMode == kScanLocal) d_topk_block(ctrl, leaves, meta, cands, p, vote.recs, vote.top_k);
    else {
      if constexpr (kExtra) d_extra_commit(ctrl, xrand, p);
      d_pick_block<kMono>(ctrl, leaves, meta, cands, p, cons.type, cons.sets_of, node.mask, forced);
    }
    if (threadIdx.x == 0) ctrl->scan_ticket = 0u;
  }
}

// The global vote and the packing of the reduced buffer, one block per packed column s = which * top_k + k, after the all-gather of every
// rank's records recs[R][2][top_k] ([UPSTREAM] VotingParallelTreeLearner::GlobalVoting).  Every block runs its leaf's vote, which is
// identical on every rank: mean = global count / R (fp32, score_t), a record's weighted gain = gain * (left_count + right_count) / mean,
// each feature keeps its largest weighted gain (strict >: the first record seen), and the top_k features by (weighted gain desc, real
// feature index asc) with a finite weighted gain are the leaf's voted features.  Block s then copies its feature's storage column of the
// leaf's LOCAL histogram (smaller: H, larger: its pool slot) into the packed buffer — of a bundle member only the member's slots, the others
// zero — and block 0 the leaves' exact local totals (LeafState::qtot).  Dynamic shared memory: 12 bytes per record of one leaf, at most
// kVoteMaxRecords records (R * top_k, checked when the booster is created).
__global__ void __launch_bounds__(256)
k_vote_pack(const TreeCtrl* __restrict__ ctrl, const LeafState* __restrict__ leaves, const FeatMeta* __restrict__ meta, const int* __restrict__ bundle_base,
            const VoteRec* __restrict__ recs, int ranks, int top_k, const long long* __restrict__ H, const long long* __restrict__ pool,
            size_t slot_elems, int* __restrict__ voted, long long* __restrict__ packed) {
  extern __shared__ double vote_ws[];
  const int n = ranks * top_k;
  double* s_wg = vote_ws;                                   // weighted gain of record i of this leaf (-inf: none)
  int* s_rf = reinterpret_cast<int*>(vote_ws + n);          // its feature, -1 after phase 2 unless it is its feature's representative
  __shared__ int s_feat;
  const int s = blockIdx.x, which = s / top_k, k = s % top_k;
  const int leaf = ctrl->go ? (which ? ctrl->larger : ctrl->smaller) : -1;
  if (threadIdx.x == 0) s_feat = -1;
  if (leaf >= 0) {
    const float mean = static_cast<float>(leaves[leaf].global_count) / static_cast<float>(ranks);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const VoteRec r = recs[(static_cast<size_t>(i / top_k) * 2 + which) * top_k + i % top_k];
      const double wg = r.gain * static_cast<double>(r.left_count + r.right_count) / static_cast<double>(mean);
      const bool ok = r.feature >= 0 && wg > kNegInf;       // -inf or NaN never beats the initial kMinScore
      s_wg[i] = ok ? wg : kNegInf; s_rf[i] = ok ? r.feature : -1;
    }
    __syncthreads();
    int rep[8];       // representative of record i = threadIdx.x + 256 j: its feature's first record with the largest weighted gain
#pragma unroll
    for (int j = 0; j < 8; ++j) rep[j] = -1;
    for (int i = threadIdx.x, j = 0; i < n; i += blockDim.x, ++j) {
      const int f = s_rf[i];
      if (f < 0) continue;
      bool first = true;
      for (int q = 0; q < n && first; ++q)
        if (q != i && s_rf[q] == f && (s_wg[q] > s_wg[i] || (s_wg[q] == s_wg[i] && q < i))) first = false;
      if (j < 8) rep[j] = first ? f : -1;
    }
    __syncthreads();
    for (int i = threadIdx.x, j = 0; i < n; i += blockDim.x, ++j) if (j < 8) s_rf[i] = rep[j];
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int f = s_rf[i];
      if (f < 0) continue;
      const int rf = meta[f].real_index;
      int rank = 0;
      for (int q = 0; q < n; ++q) {
        const int g = s_rf[q];
        if (g >= 0 && q != i && (s_wg[q] > s_wg[i] || (s_wg[q] == s_wg[i] && meta[g].real_index < rf))) ++rank;
      }
      if (rank == k) s_feat = f;
    }
  }
  __syncthreads();
  const int f = s_feat;
  if (threadIdx.x == 0) voted[s] = f;
  longlong2* dst = reinterpret_cast<longlong2*>(packed + kVoteTotals + static_cast<size_t>(s) * kVoteColumn);
  longlong2 v = make_longlong2(0, 0);
  if (f >= 0) {
    const FeatMeta fm = meta[f];
    const long long* src = (which ? pool + static_cast<size_t>(leaves[leaf].hist_slot) * slot_elems : H) + static_cast<size_t>(fm.hist_off) * 2;
    const int b = threadIdx.x, base = bundle_base ? bundle_base[f] : -1;
    if (base < 0 || (b > base && b < base + fm.num_bin)) v = reinterpret_cast<const longlong2*>(src)[b];
  }
  dst[threadIdx.x] = v;
  if (s == 0 && threadIdx.x < 2) {
    const int l = threadIdx.x ? ctrl->larger : ctrl->smaller;
    const bool has = ctrl->go && l >= 0;
    packed[2 * threadIdx.x] = has ? leaves[l].qtot[0] : 0;
    packed[2 * threadIdx.x + 1] = has ? leaves[l].qtot[1] : 0;
  }
}

// ---------------------------------------------------------------- K8/K9 leaf values -> scores
// score[row] += shrinkage * leaf_value[leaf(row)], via the final data partition
__global__ void __launch_bounds__(256)
k_add_score(const TreeCtrl* __restrict__ ctrl, const LeafState* __restrict__ leaves, TreeDev tree, const int* __restrict__ idx0,
            const int* __restrict__ idx1, double* __restrict__ score, double shrinkage) {
  const int nl = ctrl->num_leaves;
  if (nl <= 1) return;
  for (int l = 0; l < nl; ++l) {
    const LeafState& L = leaves[l];
    double v = tree.leaf_value[l] * shrinkage;
    if (!(fabs(v) > 1e-35)) v = 0.0;
    const int* src = L.buf ? idx1 : idx0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L.count; i += gridDim.x * blockDim.x) {
      const int r = L.identity ? (L.begin + i) : src[L.begin + i];
      score[r] += v;
    }
  }
}
__global__ void k_add_const(double* __restrict__ score, int n, double v) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) score[i] += v;
}
// score of a (validation) dataset += shrinkage * tree(row), traversing by bin thresholds
__global__ void __launch_bounds__(256)
k_add_tree_binned(TreeDev tree, const FeatMeta* __restrict__ meta, BinView bv, int n,
                  double* __restrict__ score, double shrinkage, double bias = 0.0, double pre_mul = 1.0, double post_mul = 1.0) {
  const int nl = *tree.num_leaves;
  if (nl <= 1) return;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int node = 0;
    while (node >= 0) {
      const int f = tree.split_feature_inner[node];
      const unsigned bin = bv.at(f, static_cast<size_t>(i));
      const int dt = tree.decision_type[node];
      bool left;
      if (dt & 1) {
        if (f >= bv.nfn) {      // wide feature: short list of bins
          left = false;
          const int len = tree.cat_list_len[node];
          for (int k = 0; k < len; ++k) left |= (bin == tree.cat_list[node * kCatListMax + k]);
        } else {
          left = (tree.cat_bits[node * 8 + (bin >> 5)] >> (bin & 31u)) & 1u;
        }
      }
      else if (((dt >> 2) & 3) == 2 && bin == static_cast<unsigned>(meta[f].num_bin - 1)) left = dt & 2;
      else left = bin <= static_cast<unsigned>(tree.threshold_bin[node]);
      node = left ? tree.left_child[node] : tree.right_child[node];
    }
    double v = tree.leaf_value[~node] * shrinkage;
    if (!(fabs(v) > 1e-35)) v = 0.0;
    score[i] = (score[i] * pre_mul + (v + bias)) * post_mul;      // rf: running average of (tree + init score); gbdt: pre = post = 1, bias = 0
  }
}
__global__ void k_scale_add(double* __restrict__ score, int n, double pre_mul, double add, double post_mul) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) score[i] = (score[i] * pre_mul + add) * post_mul;
}

// ---------------------------------------------------------------- row subsampling: bagging / GOSS  (SURVEY §8f-3)
// [LightGBM src/boosting/gbdt.cpp GBDT::BaggingHelper, goss.hpp GOSS::BaggingHelper] Rows are drawn per 1024-row block, every block
// owning an LCG (x <- 214013 x + 2531011, float = ((x >> 16) & 0x7fff) / 32768) seeded bagging_seed + block. One CUDA block per
// 1024-row block. The draw of row j of a block is the (j+1)-th LCG output, which the jump table gives directly:
// x_{j+1} = mulA[j] * x0 + addC[j], so plain bagging is embarrassingly parallel and still bit-identical to the sequential draw.
constexpr int kBagBlock = 1024;
struct LcgJump { unsigned mul[kBagBlock]; unsigned add[kBagBlock]; };

__global__ void __launch_bounds__(256)
k_bag_draw(unsigned* __restrict__ lcg_state, const LcgJump* __restrict__ jump, int n, double fraction, uint8_t* __restrict__ in_bag,
           int* __restrict__ block_count, const float* __restrict__ label = nullptr, double pos_fraction = 1.0, double neg_fraction = 1.0) {
  const int b = blockIdx.x, base = b * kBagBlock, cnt = min(kBagBlock, n - base);
  const unsigned x0 = lcg_state[b];
  int mine = 0;
  for (int j = threadIdx.x; j < cnt; j += blockDim.x) {
    const unsigned x = jump->mul[j] * x0 + jump->add[j];
    // balanced bagging (label given): positives and negatives are kept with their own fractions [LightGBM BalancedBaggingHelper]
    const double frac = label ? (label[base + j] > 0 ? pos_fraction : neg_fraction) : fraction;
    const int take = static_cast<double>(d_lcg_float(x)) < frac;
    in_bag[base + j] = static_cast<uint8_t>(take);
    mine += take;
  }
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  for (int o = 16; o; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) { block_count[b] = s_cnt; lcg_state[b] = jump->mul[cnt - 1] * x0 + jump->add[cnt - 1]; }
}

// GOSS: keep the top_rate share of rows by sum_k |g*h| and sample other_rate of the rest, amplifying the sampled gradients by
// (cnt - top_k) / other_k.  The running probability depends on how many rows were sampled so far, so the draw is sequential inside
// a 1024-row chunk (thread 0); threshold selection (bitonic sort) and the gradient scaling are parallel.
__global__ void __launch_bounds__(256)
k_goss_draw(unsigned* __restrict__ lcg_state, int n, int K, double top_rate, double other_rate, float* __restrict__ grad,
            float* __restrict__ hess, uint8_t* __restrict__ in_bag, int* __restrict__ block_count) {
  __shared__ float s_tg[kBagBlock];
  __shared__ float s_sorted[kBagBlock];
  __shared__ uint8_t s_flag[kBagBlock];      // 0 out, 1 top, 2 sampled (amplified)
  __shared__ int s_left;
  const int b = blockIdx.x, base = b * kBagBlock, cnt = min(kBagBlock, n - base);
  for (int j = threadIdx.x; j < kBagBlock; j += blockDim.x) {
    float t = -1.0f;        // padding sorts last (real values are >= 0)
    if (j < cnt) {
      t = 0.0f;
      for (int k = 0; k < K; ++k) { const size_t id = static_cast<size_t>(k) * n + base + j; t = __fadd_rn(t, fabsf(__fmul_rn(grad[id], hess[id]))); }
    }
    s_tg[j] = t; s_sorted[j] = t;
  }
  __syncthreads();
  for (int k = 2; k <= kBagBlock; k <<= 1)            // bitonic sort, descending
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < kBagBlock; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const float a = s_sorted[i], c = s_sorted[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? (a < c) : (a > c)) { s_sorted[i] = c; s_sorted[ixj] = a; }
        }
      }
      __syncthreads();
    }
  const int top_k = max(1, static_cast<int>(cnt * top_rate));
  const int other_k = static_cast<int>(cnt * other_rate);
  const float multiply = static_cast<float>(cnt - top_k) / other_k;
  if (threadIdx.x == 0) {
    const float threshold = s_sorted[top_k - 1];
    unsigned x = lcg_state[b];
    int left = 0, big = 0;
    for (int i = 0; i < cnt; ++i) {
      uint8_t f = 0;
      if (s_tg[i] >= threshold) { f = 1; ++left; ++big; }
      else {
        const int rest_need = other_k - (left - big), rest_all = (cnt - i) - (top_k - big);
        const double prob = rest_need / static_cast<double>(rest_all);
        x = 214013u * x + 2531011u;
        if (static_cast<double>(d_lcg_float(x)) < prob) { f = 2; ++left; }
      }
      s_flag[i] = f;
    }
    lcg_state[b] = x;
    s_left = left;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < cnt; j += blockDim.x) {
    const uint8_t f = s_flag[j];
    in_bag[base + j] = f ? 1 : 0;
    if (f == 2)
      for (int k = 0; k < K; ++k) { const size_t id = static_cast<size_t>(k) * n + base + j; grad[id] = __fmul_rn(grad[id], multiply); hess[id] = __fmul_rn(hess[id], multiply); }
  }
  if (threadIdx.x == 0) block_count[b] = s_left;
}

// exclusive scan of the per-block in-bag counts (single CTA), total -> *bag_total
__global__ void __launch_bounds__(1024)
k_bag_scan(int* __restrict__ block_count, int nblocks, int* __restrict__ bag_total) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < nblocks; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < nblocks ? block_count[i] : 0;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= o) incl += t; }
    if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = incl;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = s_warp[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, w, o); if (threadIdx.x >= o) w += t; }
      s_warp[threadIdx.x] = w;
    }
    __syncthreads();
    const int warp_off = (threadIdx.x >> 5) ? s_warp[(threadIdx.x >> 5) - 1] : 0;
    const int carry = s_carry;
    if (i < nblocks) block_count[i] = carry + warp_off + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + warp_off + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *bag_total = s_carry;
}
// ordered compaction: bag_idx[offset(block) + rank-in-block] = row
__global__ void __launch_bounds__(256)
k_bag_compact(const uint8_t* __restrict__ in_bag, const int* __restrict__ block_offset, int n, int* __restrict__ bag_idx) {
  __shared__ int s_warp[8];
  __shared__ int s_base;
  const int b = blockIdx.x, base = b * kBagBlock, cnt = min(kBagBlock, n - base);
  if (threadIdx.x == 0) s_base = block_offset[b];
  __syncthreads();
  for (int j0 = 0; j0 < cnt; j0 += blockDim.x) {
    const int j = j0 + threadIdx.x;
    const int take = (j < cnt) ? in_bag[base + j] : 0;
    const unsigned m = __ballot_sync(0xffffffffu, take);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int off = s_base;
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    if (take) bag_idx[off + __popc(m & ((1u << lane) - 1u))] = base + j;
    __syncthreads();
    if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < 8; ++w) t += s_warp[w]; s_base += t; }
    __syncthreads();
  }
}

// histogram int64 -> fp64 (debug / parity export)
__global__ void k_hist_to_double(const long long* __restrict__ H, double* __restrict__ out, size_t elems, const TreeCtrl* ctrl) {
  const double ig = ctrl->inv_g, ih = ctrl->inv_h;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < elems; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = static_cast<double>(H[i]) * ((i & 1) ? ih : ig);
}

}  // namespace b200gbm
