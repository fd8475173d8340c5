// Leaf-output renewal for the percentile objectives (regression_l1 / quantile / mape), SURVEY.md §8 row a9.
// Semantics restated from LightGBM v3.2.x SerialTreeLearner::RenewTreeOutput + regression_objective.hpp
// PercentileFun / WeightedPercentileFun: once a tree is grown, every leaf's output is replaced by the (weighted) alpha
// percentile of the residuals label - score of the leaf's in-bag rows.
//
// Device plan (no host round trip, the tree blob is patched in place before the score update):
//   1. k_renew_gather   : position p in the final data partition -> residual key (order-preserving u64), leaf id, row
//   2. radix sort of (key, p) over all positions, then a stable radix sort by leaf id  => rows grouped per leaf, ascending
//      residual, ties in partition order (what std::stable_sort gives upstream).  The two sorts are cub::DeviceRadixSort
//      (library code, off the hot path: it runs once per tree and only for these three objectives).
//   3. unweighted: one thread per leaf picks the two order statistics and interpolates;
//      weighted  : one CTA per leaf scans the weights into the cdf, then one thread per leaf does the upper_bound + interpolation.
//   4. data-parallel: outputs and "has rows" flags are summed over ranks (ncclAllReduce) and divided.
#pragma once
#include <cub/device/device_radix_sort.cuh>

#include "kernels.cuh"

namespace b200gbm {

__device__ __forceinline__ unsigned long long d_order_key(double x) {
  x = x + 0.0;                                          // -0.0 -> +0.0 so that equal values carry equal keys
  const long long b = __double_as_longlong(x);
  return static_cast<unsigned long long>(b) ^ (static_cast<unsigned long long>(b >> 63) | 0x8000000000000000ull);
}

// score == nullptr: residual against the constant `pred` (random forest renews against its init score)
__global__ void __launch_bounds__(256)
k_renew_gather(const TreeCtrl* __restrict__ ctrl, const LeafState* __restrict__ leaves, const int* __restrict__ idx0, const int* __restrict__ idx1,
               const float* __restrict__ label, const double* __restrict__ score, double pred, unsigned long long* __restrict__ keys,
               unsigned* __restrict__ pos_out, double* __restrict__ res_of_pos, unsigned* __restrict__ leaf_of_pos, int* __restrict__ row_of_pos) {
  const int nl = ctrl->num_leaves;
  for (int l = 0; l < nl; ++l) {
    const LeafState& L = leaves[l];
    const int* src = L.buf ? idx1 : idx0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L.count; i += gridDim.x * blockDim.x) {
      const int p = L.begin + i;
      const int r = L.identity ? p : src[p];
      const double res = static_cast<double>(label[r]) - (score ? score[r] : pred);
      keys[p] = d_order_key(res); pos_out[p] = static_cast<unsigned>(p);
      res_of_pos[p] = res; leaf_of_pos[p] = static_cast<unsigned>(l); row_of_pos[p] = r;
    }
  }
}
__global__ void k_renew_leaf_keys(const unsigned* __restrict__ sorted_pos, const unsigned* __restrict__ leaf_of_pos, int total, unsigned* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) out[i] = leaf_of_pos[sorted_pos[i]];
}
// segment starts in the leaf-grouped order: exclusive sum of the leaf counts (leaf ids ascending)
__global__ void k_renew_offsets(const TreeCtrl* __restrict__ ctrl, const LeafState* __restrict__ leaves, int* __restrict__ seg_begin) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int acc = 0;
    for (int l = 0; l < ctrl->num_leaves; ++l) { seg_begin[l] = acc; acc += leaves[l].count; }
    seg_begin[ctrl->num_leaves] = acc;
  }
}
// PercentileFun(double, residual, cnt, alpha): fp = (cnt-1)(1-alpha) in the DESCENDING order d[], interpolate d[int(fp)] .. d[int(fp)+1]
__global__ void k_renew_unweighted(const TreeCtrl* __restrict__ ctrl, const int* __restrict__ seg_begin, const unsigned* __restrict__ grouped_pos,
                                   const double* __restrict__ res_of_pos, double alpha, double* __restrict__ out, double* __restrict__ has_rows) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= ctrl->num_leaves) return;
  const int b = seg_begin[l], cnt = seg_begin[l + 1] - b;
  if (cnt <= 0) { out[l] = 0.0; has_rows[l] = 0.0; return; }
  has_rows[l] = 1.0;
  auto desc = [&](int j) { return res_of_pos[grouped_pos[b + cnt - 1 - j]]; };
  if (cnt <= 1) { out[l] = desc(0); return; }
  const double float_pos = __dmul_rn(static_cast<double>(cnt - 1), 1.0 - alpha);
  const int pos = static_cast<int>(float_pos) + 1;
  if (pos < 1) { out[l] = desc(0); return; }
  if (pos >= cnt) { out[l] = desc(cnt - 1); return; }
  const double bias = float_pos - (pos - 1);
  const double v1 = desc(pos - 1), v2 = desc(pos);
  out[l] = __dsub_rn(v1, __dmul_rn(__dsub_rn(v1, v2), bias));
}
// a + b; `inexact` is set when the sum rounds (TwoSum's error term is non-zero)
__device__ __forceinline__ double d_add_flag(double a, double b, bool& inexact) {
  const double s = __dadd_rn(a, b), bb = __dsub_rn(s, a);
  inexact |= __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb)) != 0.0;
  return s;
}
// weighted cdf per leaf: one CTA per leaf, chunked block scan with a running carry.  Upstream adds the weights one by one in row
// order.  While no add of the scan rounds (lane, warp-total and carry adds), every cdf value is the exact prefix sum, and so is every
// sequential partial sum, so the two agree.  From the first chunk in which an add rounds, the leaf's cdf is summed in row order by one
// thread, starting from the carry, which is still exact: wide weights get upstream's cdf too.
__global__ void __launch_bounds__(1024)
k_renew_cdf(const TreeCtrl* __restrict__ ctrl, const int* __restrict__ seg_begin, const unsigned* __restrict__ grouped_pos,
            const int* __restrict__ row_of_pos, const float* __restrict__ weight, double* __restrict__ cdf) {
  const int l = blockIdx.x;
  if (l >= ctrl->num_leaves) return;
  const int b = seg_begin[l], cnt = seg_begin[l + 1] - b;
  __shared__ double s_warp[32];
  __shared__ double s_v[1024];
  __shared__ double s_carry;
  if (threadIdx.x == 0) s_carry = 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  bool sequential = false;      // the same in every thread of the block
  for (int base = 0; base < cnt; base += 1024) {
    const int i = base + threadIdx.x;
    const double v = i < cnt ? static_cast<double>(weight[row_of_pos[grouped_pos[b + i]]]) : 0.0;
    if (!sequential) {
      bool inexact = false;
      double incl = v;
      for (int o = 1; o < 32; o <<= 1) { const double t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl = d_add_flag(incl, t, inexact); }
      if (lane == 31) s_warp[warp] = incl;
      __syncthreads();
      if (warp == 0) {
        double w = s_warp[lane];
        for (int o = 1; o < 32; o <<= 1) { const double t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w = d_add_flag(w, t, inexact); }
        s_warp[lane] = w;
      }
      __syncthreads();
      const double carry = s_carry, woff = warp ? s_warp[warp - 1] : 0.0;
      const double c = d_add_flag(carry, d_add_flag(woff, incl, inexact), inexact);
      sequential = __syncthreads_or(inexact);
      if (!sequential) {
        if (i < cnt) cdf[b + i] = c;
        if (threadIdx.x == 1023) s_carry = c;
      }
      __syncthreads();
    }
    if (sequential) {
      s_v[threadIdx.x] = v;
      __syncthreads();
      if (threadIdx.x == 0) {
        double c = s_carry;
        for (int j = 0, m = min(1024, cnt - base); j < m; ++j) { c = __dadd_rn(c, s_v[j]); cdf[b + base + j] = c; }
        s_carry = c;
      }
      __syncthreads();
    }
  }
}
// WeightedPercentileFun(double, residual, weight, cnt, alpha) on the ascending order
__global__ void k_renew_weighted(const TreeCtrl* __restrict__ ctrl, const int* __restrict__ seg_begin, const unsigned* __restrict__ grouped_pos,
                                 const double* __restrict__ res_of_pos, const double* __restrict__ cdf, double alpha, double* __restrict__ out,
                                 double* __restrict__ has_rows) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= ctrl->num_leaves) return;
  const int b = seg_begin[l], cnt = seg_begin[l + 1] - b;
  if (cnt <= 0) { out[l] = 0.0; has_rows[l] = 0.0; return; }
  has_rows[l] = 1.0;
  auto asc = [&](int j) { return res_of_pos[grouped_pos[b + j]]; };
  if (cnt <= 1) { out[l] = asc(0); return; }
  const double* c = cdf + b;
  const double threshold = __dmul_rn(c[cnt - 1], alpha);
  int lo = 0, hi = cnt;                       // upper_bound: first index with cdf > threshold
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (c[mid] > threshold) hi = mid; else lo = mid + 1; }
  int pos = min(lo, cnt - 1);
  if (pos == 0 || pos == cnt - 1) { out[l] = asc(pos); return; }
  const double v1 = asc(pos - 1), v2 = asc(pos);
  const double step = __dsub_rn(c[pos + 1], c[pos]);
  if (step >= 1.0) out[l] = __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn(threshold, c[pos]), step), __dsub_rn(v2, v1)), v1);
  else out[l] = v2;
}
// leaf_value[l] = out[l] / max(1, workers[l]) (workers == 1 on a single rank)
__global__ void k_renew_apply(const TreeCtrl* __restrict__ ctrl, TreeDev tree, const double* __restrict__ out, const double* __restrict__ has_rows, int parallel) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= ctrl->num_leaves || ctrl->num_leaves <= 1) return;
  tree.leaf_value[l] = parallel ? (has_rows[l] > 0.0 ? out[l] / has_rows[l] : 0.0) : out[l];
}

}  // namespace b200gbm
