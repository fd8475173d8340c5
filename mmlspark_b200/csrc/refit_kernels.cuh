// Kernels of LGBM_BoosterRefit (refit.cu): the leaf-index staging, the per-leaf sums, the leaf rule and the score update.
// Semantics restated from LightGBM v3.2.x GBDT::RefitTree + SerialTreeLearner::FitByExistingTree, from knowledge.
#pragma once
#include "bin_mapper.h"      // kZeroThr
#include "kernels.cuh"

namespace b200gbm {

// One row block of leaf_preds, [rows][mb] (the batch's models m0 .. m0 + mb - 1 of rows r0 .. r0 + rows - 1), into per-model leaf
// columns cols[j][row] (n rows each), through a 32 x 32 shared tile so that both the read and the write are coalesced.  Every index
// outside [0, num_leaves of its model) lowers first_bad to its position row * ncol + model in the caller's row-major matrix, so the
// smallest one left is the first bad (row, model).  grid: x over 32-row tiles, y over 32-model tiles; block 32 x 8.
__global__ void __launch_bounds__(256)
k_refit_stage(const int* __restrict__ block, int rows, int mb, long long r0, int n, int m0, int ncol, const int* __restrict__ num_leaves,
              int* __restrict__ cols, unsigned long long* __restrict__ first_bad) {
  __shared__ int tile[32][33];
  const int i0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  const int j = j0 + threadIdx.x;
  const int limit = j < mb ? num_leaves[m0 + j] : 0;
  for (int dy = threadIdx.y; dy < 32; dy += 8) {
    const int i = i0 + dy;
    if (i < rows && j < mb) {
      const int v = block[static_cast<size_t>(i) * mb + j];
      tile[dy][threadIdx.x] = v;
      if (v < 0 || v >= limit) atomicMin(first_bad, static_cast<unsigned long long>((r0 + i) * ncol + m0 + j));
    }
  }
  __syncthreads();
  const int i = i0 + threadIdx.x;
  for (int dy = threadIdx.y; dy < 32; dy += 8)
    if (i < rows && j0 + dy < mb) cols[static_cast<size_t>(j0 + dy) * n + r0 + i] = tile[threadIdx.x][dy];
}

// Per-leaf sums of one tree: sums[l] = sum q_g, sums[L + l] = sum q_h, sums[2L + l] = rows, over the rows whose leaf is l, with q on
// K3's 36-bit fixed-point grid (d_fixed at k_set_scale's exponents).  Integer sums are exact and order-free, so any grid and any split
// of the rows over ranks give the same bits.  Constant hessians leave the q_h plane alone: the count plane is their sum, as in k_quantize.
// kShared: every CTA adds into its own copy of the 3 x L sums in shared memory (L <= kRefitSharedLeaves) and adds the copy to `sums`
// once; otherwise every row adds into `sums` with global atomics.  sums: zeroed.
constexpr int kRefitSharedLeaves = 4096;      // 3 x 4096 x 8 B = 96 KB of shared memory per CTA
template <bool kShared>
__global__ void __launch_bounds__(256)
k_refit_leaf_sums(const int* __restrict__ leaf, const float* __restrict__ g, const float* __restrict__ h, int n, int num_leaves,
                  int const_hessian, const TreeCtrl* __restrict__ ctrl, long long* __restrict__ sums) {
  extern __shared__ long long s_sums[];
  const int eg = ctrl->exp_g, eh = ctrl->exp_h;
  unsigned long long* acc = reinterpret_cast<unsigned long long*>(kShared ? s_sums : sums);
  if (kShared) {
    for (int l = threadIdx.x; l < 3 * num_leaves; l += blockDim.x) s_sums[l] = 0;
    __syncthreads();
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int l = leaf[i];
    atomicAdd(&acc[l], static_cast<unsigned long long>(d_fixed(g[i], eg)));
    if (!const_hessian) atomicAdd(&acc[num_leaves + l], static_cast<unsigned long long>(d_fixed(h[i], eh)));
    atomicAdd(&acc[2 * num_leaves + l], 1ull);
  }
  if (kShared) {
    __syncthreads();
    for (int l = threadIdx.x; l < 3 * num_leaves; l += blockDim.x)
      if (s_sums[l]) atomicAdd(reinterpret_cast<unsigned long long*>(&sums[l]), static_cast<unsigned long long>(s_sums[l]));
  }
}

// One thread per leaf: FitByExistingTree's rule at the (all-reduced) sums.
//   sum_g = Q_g 2^-e_g, sum_h = kEpsilon + Q_h 2^-e_h (constant hessians: kEpsilon + count), cnt = rows;
//   output = CalculateSplittedLeafOutput(sum_g, sum_h, l1, l2, max_delta_step), unconstrained; with path smoothing and l > 0 it is
//            smoothed with cnt rows toward leaf_parent[l] itself: upstream passes the parent's node index where a parent output is
//            expected, and this restates that.  A leaf no row reaches gets output 0.
//   leaf = MaybeRoundToZero(decay * leaf + (1 - decay) * output * shrinkage), in that order of fp64 operations (no contraction).
__global__ void k_refit_apply(const long long* __restrict__ sums, int num_leaves, const TreeCtrl* __restrict__ ctrl, int const_hessian,
                              const double* __restrict__ old_leaf, const int* __restrict__ leaf_parent, double shrinkage, double decay,
                              SplitParams p, double* __restrict__ new_leaf) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= num_leaves) return;
  const long long cnt = sums[2 * num_leaves + l];
  double out = 0.0;
  if (cnt > 0) {
    const double sg = static_cast<double>(sums[l]) * ldexp(1.0, -ctrl->exp_g);
    const double sh = kPathSmoothEps + (const_hessian ? static_cast<double>(cnt) : static_cast<double>(sums[num_leaves + l]) * ldexp(1.0, -ctrl->exp_h));
    SplitParams q = p;
    if (l == 0) q.path_smooth = 0.0;
    out = d_smooth_output(sg, sh, static_cast<int>(cnt), static_cast<double>(leaf_parent[l]), q);
  }
  const double v = __dadd_rn(__dmul_rn(decay, old_leaf[l]), __dmul_rn(1.0 - decay, __dmul_rn(out, shrinkage)));
  new_leaf[l] = fabs(v) > kZeroThr ? v : 0.0;
}

// score[row] += the refit tree's value at the row's leaf
__global__ void __launch_bounds__(256)
k_refit_add_score(const int* __restrict__ leaf, const double* __restrict__ value, int n, double* __restrict__ score) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) score[i] += value[leaf[i]];
}

}  // namespace b200gbm
