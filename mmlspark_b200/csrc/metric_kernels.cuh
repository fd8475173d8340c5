// Evaluation metrics on the device (LGBM_BoosterGetEval, reference call sites TrainUtils.scala:125-151 and
// LightGBMBooster.scala:296-310).  Round 1 downloaded all K*n fp64 scores and looped on one host thread (0.8 GB per call at 100M rows);
// here every metric is a reduction over the device-resident scores and only a handful of doubles cross PCIe.
//   point-wise losses  [UPSTREAM regression_metric.hpp / binary_metric.hpp / multiclass_metric.hpp / xentropy_metric.hpp]:
//                      k_metric_pointwise -> per-block partial sums -> k_metric_finish (fixed summation order: reproducible)
//   auc                [UPSTREAM binary_metric.hpp AUCMetric]: radix sort by score (cub, library code off the training path), prefix sums of
//                      the positive / negative weights, one term per group of tied scores
//   average_precision  [UPSTREAM binary_metric.hpp AveragePrecisionMetric]: the same sort and prefix sums as auc, one term per tie group
//                      holding positives: its positive weight times the precision through the group
//   auc_mu             [UPSTREAM multiclass_metric.hpp AucMuMetric]: rows grouped by class (stable radix sort by label), then batches of
//                      class pairs of about 2n items: per pair a segment of (key of the pair's distance d, row) for the rows of both
//                      classes, a segmented sort (a device-wide radix sort for each large segment), segmented prefix sums and the auc
//                      terms per segment; scratch stays O(n) for any K
//   ndcg@k / map@k     [UPSTREAM rank_metric.hpp, dcg_calculator.cpp, map_metric.hpp]: one block per query, stable rank by counting
// Every sum of non-integer terms runs in a fixed order (contiguous row ranges per block, blocks summed in block order), so repeated
// evaluations are bit-identical.
#pragma once
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include <cstdint>

namespace b200gbm {

enum MetricKind {
  kMetL2 = 0, kMetL1, kMetHuber, kMetFair, kMetPoisson, kMetGamma, kMetTweedie, kMetQuantile, kMetMape, kMetBinLogloss, kMetBinError,
  kMetMultiLogloss, kMetMultiError, kMetXent, kMetGammaDeviance, kMetXentLambda, kMetKLDiv
};
struct MetricParams {
  int kind, K, ova;
  int transform;               // the objective's single-output transform (HostModel::ObjectiveTransform kind) and its sigmoid,
  double alpha, fair_c, rho, sigmoid;
  double transform_sigmoid;    // for cross_entropy_lambda and kullback_leibler
};

// [UPSTREAM xentropy_metric.hpp XentLoss / YentLoss]: log arguments clipped at 1e-12; YentLoss is minus the label's entropy, so that
// kullback_leibler = mean XentLoss + mean YentLoss is 0 where p equals the label
__device__ __forceinline__ double d_xent_loss(double lab, double p) {
  const double a = lab * (p > 1e-12 ? log(p) : log(1e-12)), b = (1.0 - lab) * (1.0 - p > 1e-12 ? log(1.0 - p) : log(1e-12));
  return -(a + b);
}
__device__ __forceinline__ double d_yent_loss(double p) {
  double hp = 0.0;
  if (p > 1e-12) hp += p * log(p);
  const double q = 1.0 - p;
  if (q > 1e-12) hp += q * log(q);
  return hp;
}
// single-output transforms of HostModel::ConvertScores
__device__ __forceinline__ double d_output_transform(int kind, double sigmoid, double x) {
  switch (kind) {
    case 1: return 1.0 / (1.0 + exp(-sigmoid * x));
    case 3: return exp(x);
    case 5: return log1p(exp(x));
    case 6: return (x >= 0 ? 1.0 : -1.0) * x * x;
    default: return x;
  }
}

// loss of one row; score = class-major raw scores, w = the row's weight (only cross_entropy_lambda reads it)
__device__ __forceinline__ double d_point_loss(const MetricParams& mp, const double* __restrict__ score, size_t n, size_t i, double lab, double w) {
  const double eps = 1e-15;
  double s0 = score[i];
  switch (mp.kind) {
    case kMetL2: { const double d = s0 - lab; return d * d; }
    case kMetL1: return fabs(s0 - lab);
    case kMetHuber: { const double d = s0 - lab; return fabs(d) <= mp.alpha ? 0.5 * d * d : mp.alpha * (fabs(d) - 0.5 * mp.alpha); }
    case kMetFair: { const double x = fabs(s0 - lab), c = mp.fair_c; return c * x - c * c * log(1.0 + x / c); }
    case kMetPoisson: { double sc = exp(s0); sc = fmax(sc, 1e-10); return sc - lab * log(sc); }
    case kMetGamma: {
      const double sc = exp(s0), theta = -1.0 / sc, b = -(-theta > 0 ? log(-theta) : -INFINITY);
      const double ll = lab > 0 ? log(lab) : -INFINITY, cc = ll - ll;      // psi = 1: (1/psi) log(label/psi) - log(label) - lgamma(1/psi)
      return -((lab * theta - b) + cc);
    }
    case kMetGammaDeviance: { const double sc = exp(s0), tmp = lab / (sc + 1e-9); return tmp - (tmp > 0 ? log(tmp) : -INFINITY) - 1; }
    case kMetTweedie: {
      double sc = fmax(exp(s0), 1e-10);
      const double rho = mp.rho;
      return -lab * exp((1 - rho) * log(sc)) / (1 - rho) + exp((2 - rho) * log(sc)) / (2 - rho);
    }
    case kMetQuantile: { const double delta = lab - s0; return delta < 0 ? (mp.alpha - 1.0) * delta : mp.alpha * delta; }
    case kMetMape: return fabs(lab - s0) / fmax(1.0, fabs(lab));
    case kMetBinLogloss: case kMetBinError: {
      const double p = 1.0 / (1.0 + exp(-mp.sigmoid * s0));
      if (mp.kind == kMetBinError) return ((p <= 0.5) == (lab > 0)) ? 1.0 : 0.0;
      const double pl = lab > 0 ? p : 1.0 - p;
      return pl > eps ? -log(pl) : -log(eps);
    }
    case kMetXent: return d_xent_loss(lab, 1.0 / (1.0 + exp(-s0)));
    case kMetXentLambda: return d_xent_loss(lab, 1.0 - exp(-w * d_output_transform(mp.transform, mp.transform_sigmoid, s0)));
    case kMetKLDiv: return d_yent_loss(lab) + d_xent_loss(lab, d_output_transform(mp.transform, mp.transform_sigmoid, s0));
    case kMetMultiLogloss: case kMetMultiError: {
      // probabilities by the objective's ConvertOutput: softmax, or a sigmoid per class for multiclassova
      const int K = mp.K, l = static_cast<int>(lab);
      double pl = 0.0;
      int larger = 0;
      if (mp.ova) {
        pl = 1.0 / (1.0 + exp(-mp.sigmoid * score[static_cast<size_t>(l) * n + i]));
        if (mp.kind == kMetMultiError)
          for (int k = 0; k < K; ++k) larger += (1.0 / (1.0 + exp(-mp.sigmoid * score[static_cast<size_t>(k) * n + i]))) >= pl;
      } else {
        double mx = s0;
        for (int k = 1; k < K; ++k) mx = fmax(mx, score[static_cast<size_t>(k) * n + i]);
        double sum = 0;
        for (int k = 0; k < K; ++k) sum += exp(score[static_cast<size_t>(k) * n + i] - mx);
        pl = exp(score[static_cast<size_t>(l) * n + i] - mx) / sum;
        if (mp.kind == kMetMultiError)
          for (int k = 0; k < K; ++k) larger += (exp(score[static_cast<size_t>(k) * n + i] - mx) / sum) >= pl;
      }
      if (mp.kind == kMetMultiError) return larger > 1 ? 1.0 : 0.0;
      return pl > eps ? -log(pl) : -log(eps);
    }
  }
  return 0.0;
}

constexpr int kMetricBlock = 256;
__device__ __forceinline__ void d_block_sum2(double& a, double& b, double* sm /*[2*8]*/) {
  for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { sm[warp] = a; sm[8 + warp] = b; }
  __syncthreads();
  if (threadIdx.x == 0) { a = 0; b = 0; for (int w = 0; w < kMetricBlock / 32; ++w) { a += sm[w]; b += sm[8 + w]; } }
}
__global__ void __launch_bounds__(kMetricBlock)
k_metric_pointwise(const double* __restrict__ score, const float* __restrict__ label, const float* __restrict__ weight, int n, MetricParams mp,
                   double* __restrict__ partial) {
  __shared__ double sm[16];
  double loss = 0, sw = 0;
  // contiguous row ranges per block and a fixed thread stride: the summation order does not depend on the grid schedule
  const long long per = (static_cast<long long>(n) + gridDim.x - 1) / gridDim.x;
  const long long r0 = per * blockIdx.x, r1 = min(r0 + per, static_cast<long long>(n));
  for (long long i = r0 + threadIdx.x; i < r1; i += kMetricBlock) {
    const double w = weight ? static_cast<double>(weight[i]) : 1.0;
    const double rw = mp.kind == kMetXentLambda ? 1.0 : w;      // [UPSTREAM] cross_entropy_lambda: w is inside the loss, the mean is over rows
    loss += d_point_loss(mp, score, static_cast<size_t>(n), static_cast<size_t>(i), static_cast<double>(label[i]), w) * rw;
    sw += rw;
  }
  d_block_sum2(loss, sw, sm);
  if (threadIdx.x == 0) { partial[2 * blockIdx.x] = loss; partial[2 * blockIdx.x + 1] = sw; }
}
// out[c] = sum over blocks of partial[b * stride + c], c < stride <= 32: one warp, lane = column, sequential over blocks
__global__ void k_metric_finish(const double* __restrict__ partial, int blocks, int stride, double* __restrict__ out) {
  const int c = threadIdx.x;
  if (c >= stride) return;
  double s = 0;
  for (int b = 0; b < blocks; ++b) s += partial[static_cast<size_t>(b) * stride + c];
  out[c] = s;
}

// ---------------------------------------------------------------- AUC
__device__ __forceinline__ unsigned long long d_sortable(double v) {
  unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(v));
  return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
}
// -0.0 is keyed as +0.0: the two compare equal, so they are one tie group, as in [UPSTREAM AUCMetric] `cur_score != threshold` and in
// scikit-learn's roc_auc_score (an init_score can hold -0.0)
__global__ void k_auc_keys(const double* __restrict__ score, int n, unsigned long long* __restrict__ keys, int* __restrict__ rows) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double s = score[i];
    keys[i] = d_sortable(s == 0.0 ? 0.0 : s); rows[i] = i;
  }
}
// sorted position i (descending score): weights of the row split by class, and the head marker of its tie group
__global__ void k_auc_weights(const unsigned long long* __restrict__ keys, const int* __restrict__ rows, const float* __restrict__ label,
                              const float* __restrict__ weight, int n, double* __restrict__ wpos, double* __restrict__ wneg, int* __restrict__ head) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int r = rows[i];
    const double w = weight ? static_cast<double>(weight[r]) : 1.0;
    const bool pos = label[r] > 0;
    wpos[i] = pos ? w : 0.0; wneg[i] = pos ? 0.0 : w;
    head[i] = (i == 0 || keys[i] != keys[i - 1]) ? i : 0;
  }
}
// one term per tie group, taken at the group's last position t: neg_g * (pos_g / 2 + positives ranked strictly above)
__global__ void __launch_bounds__(kMetricBlock)
k_auc_terms(const unsigned long long* __restrict__ keys, const int* __restrict__ start, const double* __restrict__ ppos, const double* __restrict__ pneg,
            int n, double* __restrict__ partial) {
  __shared__ double sm[16];
  double acc = 0, unused = 0;
  const long long per = (static_cast<long long>(n) + gridDim.x - 1) / gridDim.x;
  const long long r0 = per * blockIdx.x, r1 = min(r0 + per, static_cast<long long>(n));
  for (long long t = r0 + threadIdx.x; t < r1; t += kMetricBlock) {
    if (t != n - 1 && keys[t] == keys[t + 1]) continue;
    const int s = start[t];
    const double before_p = s > 0 ? ppos[s - 1] : 0.0, before_n = s > 0 ? pneg[s - 1] : 0.0;
    const double pos_g = ppos[t] - before_p, neg_g = pneg[t] - before_n;
    acc += neg_g * (pos_g * 0.5 + before_p);
  }
  d_block_sum2(acc, unused, sm);
  if (threadIdx.x == 0) { partial[2 * blockIdx.x] = acc; partial[2 * blockIdx.x + 1] = 0.0; }
}

// ---------------------------------------------------------------- average_precision
// after the auc sort and prefix sums: one term per tie group, at its last position t, pos_g * TP / (TP + FP) with TP / FP the positive /
// negative weight ranked at or above the group.  A group without positive weight adds nothing (no 0/0 on zero-weight groups).
__global__ void __launch_bounds__(kMetricBlock)
k_ap_terms(const unsigned long long* __restrict__ keys, const int* __restrict__ start, const double* __restrict__ ppos, const double* __restrict__ pneg,
           int n, double* __restrict__ partial) {
  __shared__ double sm[16];
  double acc = 0, unused = 0;
  const long long per = (static_cast<long long>(n) + gridDim.x - 1) / gridDim.x;
  const long long r0 = per * blockIdx.x, r1 = min(r0 + per, static_cast<long long>(n));
  for (long long t = r0 + threadIdx.x; t < r1; t += kMetricBlock) {
    if (t != n - 1 && keys[t] == keys[t + 1]) continue;
    const int s = start[t];
    const double tp = ppos[t], fp = pneg[t], pos_g = tp - (s > 0 ? ppos[s - 1] : 0.0);
    if (pos_g != 0.0) acc += pos_g * __drcp_rn(tp + fp) * tp;      // a reciprocal: the IEEE division's slow path would spill
  }
  d_block_sum2(acc, unused, sm);
  if (threadIdx.x == 0) { partial[2 * blockIdx.x] = acc; partial[2 * blockIdx.x + 1] = 0.0; }
}

// ---------------------------------------------------------------- auc_mu
// class-grouped row order: key = the row's class (labels are checked to lie in [0, K)), sorted stably by cub's radix sort
__global__ void k_class_keys(const float* __restrict__ label, int n, unsigned* __restrict__ keys, int* __restrict__ rows) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    keys[i] = static_cast<unsigned>(static_cast<int>(label[i])); rows[i] = i;
  }
}
// cls_start[c] = first position of class c in the sorted keys, cls_start[K] = n; an absent class gets an empty range.  The host zeroes
// cls_start first, which is the answer for n = 0.
__global__ void k_class_bounds(const unsigned* __restrict__ keys, int n, int K, int* __restrict__ cls_start) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int c = static_cast<int>(keys[i]), prev = i == 0 ? -1 : static_cast<int>(keys[i - 1]);
    for (int k = prev + 1; k <= c; ++k) cls_start[k] = i;
    if (i == n - 1) for (int k = c + 1; k <= K; ++k) cls_start[k] = n;
  }
}
// the segment g of batch item q: the largest g with off[g] <= q (empty segments share their offset with the next one)
__device__ __forceinline__ int d_segment_of(const int* __restrict__ off, int P, long long q) {
  int lo = 0, hi = P - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (off[mid] <= q) lo = mid; else hi = mid - 1; }
  return lo;
}
// One batch of class pairs [p0, p0 + P): segment g holds the rows of pair p0 + g = (i, j), first class i's rows, then class j's, and
// spans items [off[g], off[g + 1]).  pv[p] = (t1, v[0..K)) for pair p; every row gets d = t1 * sum_c v[c] * s_c over the raw class-major
// scores (a zero v[c] adds nothing, so the default matrix reads two scores per row).  -0.0 is keyed as +0.0, as in k_auc_keys.
__global__ void k_aucmu_keys(const double* __restrict__ score, int n, int K, const int* __restrict__ cls_start, const int* __restrict__ cls_rows,
                             const int2* __restrict__ pairs, const double* __restrict__ pv, int p0, int P, const int* __restrict__ off,
                             unsigned long long* __restrict__ keys, int* __restrict__ rows, int* __restrict__ seg) {
  const int N = off[P];
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < N; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = d_segment_of(off, P, q);
    const int2 pr = pairs[p0 + g];
    const int local = static_cast<int>(q - off[g]), ni = cls_start[pr.x + 1] - cls_start[pr.x];
    const int r = local < ni ? cls_rows[cls_start[pr.x] + local] : cls_rows[cls_start[pr.y] + local - ni];
    const double* v = pv + static_cast<size_t>(p0 + g) * (K + 1);
    double dot = 0.0;
    for (int c = 0; c < K; ++c) {
      const double vc = v[1 + c];
      if (vc != 0.0) dot += vc * score[static_cast<size_t>(c) * n + r];
    }
    const double d = v[0] * dot;
    keys[q] = d_sortable(d == 0.0 ? 0.0 : d); rows[q] = r; seg[q] = g;
  }
}
// sorted batch position q (descending d within its segment): the row's weight as class i ("positive") or class j, and the head marker of
// its tie group; a segment's first position is always a head, so the max-scan of the heads never reaches into the previous segment
__global__ void k_aucmu_weights(const unsigned long long* __restrict__ keys, const int* __restrict__ rows, const int* __restrict__ seg,
                                const int* __restrict__ off, const int2* __restrict__ pairs, int p0, const float* __restrict__ label,
                                const float* __restrict__ weight, int N, double* __restrict__ wpos, double* __restrict__ wneg, int* __restrict__ head) {
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < N; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = seg[q], r = rows[q];
    const double w = weight ? static_cast<double>(weight[r]) : 1.0;
    const bool pos = static_cast<int>(label[r]) == pairs[p0 + g].x;
    wpos[q] = pos ? w : 0.0; wneg[q] = pos ? 0.0 : w;
    head[q] = (q == off[g] || keys[q] != keys[q - 1]) ? q : 0;
  }
}
// k_auc_terms per segment, over the segmented prefix sums: each block takes a contiguous range of the batch's items and reduces once
// per segment its range touches into partial[block * P + g] (the host zeroes the rest)
__global__ void __launch_bounds__(kMetricBlock)
k_aucmu_terms(const unsigned long long* __restrict__ keys, const int* __restrict__ start, const double* __restrict__ ppos, const double* __restrict__ pneg,
              const int* __restrict__ off, int P, double* __restrict__ partial) {
  __shared__ double sm[16];
  const long long N = off[P];
  const long long per = (N + gridDim.x - 1) / gridDim.x;
  const long long r0 = per * blockIdx.x, r1 = min(r0 + per, N);
  if (r0 >= r1) return;
  for (int g = d_segment_of(off, P, r0); g < P && off[g] < r1; ++g) {
    const long long sb = off[g], se = off[g + 1], a = max(r0, sb), b = min(r1, se);
    double acc = 0, unused = 0;
    for (long long t = a + threadIdx.x; t < b; t += kMetricBlock) {
      if (t != se - 1 && keys[t] == keys[t + 1]) continue;
      const int s = start[t];
      const double before_p = s > sb ? ppos[s - 1] : 0.0, before_n = s > sb ? pneg[s - 1] : 0.0;
      const double pos_g = ppos[t] - before_p, neg_g = pneg[t] - before_n;
      acc += neg_g * (pos_g * 0.5 + before_p);
    }
    d_block_sum2(acc, unused, sm);
    if (threadIdx.x == 0) partial[static_cast<size_t>(blockIdx.x) * P + g] = acc;
    __syncthreads();      // sm is reused by the next segment
  }
}
// S[p0 + g] = AUC of pair g: its block partials summed in block order, over W_i * W_j (the class weights are the segment's last prefix
// sums).  A class without rows or weight gives 0 / 0 = NaN, as upstream does not guard that division.
__global__ void k_aucmu_pair_finish(const double* __restrict__ partial, int blocks, int P, const int* __restrict__ off, const double* __restrict__ ppos,
                                    const double* __restrict__ pneg, int p0, double* __restrict__ S) {
  for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < P; g += gridDim.x * blockDim.x) {
    double s = 0;
    for (int b = 0; b < blocks; ++b) s += partial[static_cast<size_t>(b) * P + g];
    const int e = off[g + 1];
    const bool any = e > off[g];
    const double wi = any ? ppos[e - 1] : 0.0, wj = any ? pneg[e - 1] : 0.0;
    S[p0 + g] = s / (wi * wj);
  }
}
// auc_mu = 2 / (K (K - 1)) * sum of the pairs' AUCs, summed in pair order by one thread
__global__ void k_aucmu_total(const double* __restrict__ S, int npairs, int K, double* __restrict__ out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  double s = 0;
  for (int p = 0; p < npairs; ++p) s += S[p];
  out[0] = s * (2.0 / (static_cast<double>(K) * (K - 1)));
}

// ---------------------------------------------------------------- ndcg@k / map@k : one block per query
// out partial[q_block][2 * nk]: ndcg sums then map sums for the nk cut-offs (ks ascending as the reference sorts eval_at)
constexpr int kMaxEvalAt = 16;
struct RankEvalParams { int nk; int ks[kMaxEvalAt]; int want_ndcg, want_map; };
__global__ void __launch_bounds__(128)
k_metric_rank(const double* __restrict__ score, const float* __restrict__ label, const int* __restrict__ qb, int nq, const double* __restrict__ label_gain,
              int num_gain, const double* __restrict__ discount, RankEvalParams rp, int max_q, double* __restrict__ partial) {
  extern __shared__ unsigned char rk_smem[];
  double* r_score = reinterpret_cast<double*>(rk_smem);          // [max_q] document order
  int* s_lab = reinterpret_cast<int*>(r_score + max_q);          // [max_q] label by sorted position
  float* r_lab = reinterpret_cast<float*>(s_lab + max_q);        // [max_q] label in document order
  __shared__ int s_cnt[64];                                      // label value histogram (label_gain has <= 31 entries by default)
  double acc[2 * kMaxEvalAt];
  for (int k = 0; k < 2 * kMaxEvalAt; ++k) acc[k] = 0.0;
  const long long per = (static_cast<long long>(nq) + gridDim.x - 1) / gridDim.x;
  const long long q0 = per * blockIdx.x, q1 = min(q0 + per, static_cast<long long>(nq));
  for (long long q = q0; q < q1; ++q) {
    const int start = qb[q], cnt = qb[q + 1] - start;
    __syncthreads();
    if (threadIdx.x < 64) s_cnt[threadIdx.x] = 0;
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) { r_score[i] = score[start + i]; r_lab[i] = label[start + i]; }
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const double si = r_score[i];
      int rank = 0;
      for (int j = 0; j < cnt; ++j) { const double sj = r_score[j]; rank += (sj > si) || (sj == si && j < i); }
      const int li = static_cast<int>(r_lab[i]);
      s_lab[rank] = r_lab[i] > 0.5f ? (li | 0x40000000) : li;       // bit 30: "relevant" for MAP (label > 0.5)
      if (li >= 0 && li < 64) atomicAdd(&s_cnt[li], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (rp.want_ndcg) {
        // [UPSTREAM DCGCalculator::CalMaxDCG] then CalDCG, both sequential in position order
        double maxdcg[kMaxEvalAt];
        {
          int top = num_gain - 1, left = 0;
          double cur = 0;
          int lc[64];
          for (int v = 0; v < 64; ++v) lc[v] = s_cnt[v];
          for (int e = 0; e < rp.nk; ++e) {
            const int ck = min(rp.ks[e], cnt);
            for (int j = left; j < ck; ++j) {
              while (top > 0 && lc[top] <= 0) --top;
              if (top < 0) break;
              cur += discount[j] * label_gain[top];
              --lc[top];
            }
            maxdcg[e] = cur;
            left = ck;
          }
        }
        if (!(maxdcg[0] > 0.0)) {
          for (int e = 0; e < rp.nk; ++e) acc[e] += 1.0;
        } else {
          double cur = 0;
          int left = 0;
          for (int e = 0; e < rp.nk; ++e) {
            const int ck = min(rp.ks[e], cnt);
            for (int j = left; j < ck; ++j) cur += label_gain[s_lab[j] & 0x3fffffff] * discount[j];
            acc[e] += cur * (1.0 / maxdcg[e]);
            left = ck;
          }
        }
      }
      if (rp.want_map) {
        // [UPSTREAM MapMetric::CalMapAtK]
        int npos = 0;
        for (int j = 0; j < cnt; ++j) npos += (s_lab[j] >> 30) & 1;
        int num_hit = 0, left = 0;
        double sum_ap = 0;
        for (int e = 0; e < rp.nk; ++e) {
          const int ck = min(rp.ks[e], cnt);
          for (int j = left; j < ck; ++j)
            if ((s_lab[j] >> 30) & 1) { ++num_hit; sum_ap += num_hit / (j + 1.0f); }
          acc[kMaxEvalAt + e] += npos > 0 ? sum_ap / min(npos, ck) : 1.0;
          left = ck;
        }
      }
    }
  }
  if (threadIdx.x == 0)
    for (int k = 0; k < 2 * kMaxEvalAt; ++k) partial[static_cast<size_t>(blockIdx.x) * 2 * kMaxEvalAt + k] = acc[k];
}

}  // namespace b200gbm
