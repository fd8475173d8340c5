// Batched prediction kernels of the Predictor (predictor.h): the flattened forest's tree walk, the raw-score, leaf-index and TreeSHAP
// kernels over dense rows, and the two kernels that read CSR rows through a dense row of slots.
#pragma once
#include <cuda_runtime.h>

namespace b200gbm {

// ---------------------------------------------------------------- batched prediction (SURVEY §8f-2)
// Flattened forest on the device; one thread per (row, class) walks the trees of its class in model order, so the raw
// score is the same sequence of fp64 additions as the host predictor (HostModel::PredictRow) => bit-identical.
struct ForestDev {
  const int* tree_offset;        // [num_trees+1] node offset of each tree (a tree with L leaves has L-1 nodes)
  const int* leaf_offset;        // [num_trees+1]
  const int* num_leaves;         // [num_trees]
  const int* split_feature;      // per node: real feature index
  const double* threshold;
  const int* decision_type;
  const int* left_child;
  const int* right_child;
  const double* leaf_value;
  const int* cat_begin;          // per node: categorical nodes index their category bitset in cat_words
  const int* cat_len;
  const unsigned* cat_words;
  const double* node_count;      // per node: rows that reached it in training (TreeSHAP cover)
  const double* leaf_count;      // per leaf
  const double* expected;        // per tree: count-weighted mean leaf value
};
// child of global node g for this row (Tree::Decision: numerical with missing handling, or categorical bitset)
template <typename T>
__device__ __forceinline__ int d_node_child(const ForestDev& f, int g, const T* __restrict__ row) {
  double fval = static_cast<double>(row[f.split_feature[g]]);
  const int dt = f.decision_type[g];
  const int mt = (dt >> 2) & 3;
  bool left;
  if (dt & 1) {                 // categorical decision: NaN goes right whatever the missing type (HostTree::Decide)
    left = false;
    if (!isnan(fval)) {
      const int iv = static_cast<int>(fval);
      const int w = iv >> 5;
      if (iv >= 0 && w < f.cat_len[g]) left = (f.cat_words[f.cat_begin[g] + w] >> (iv & 31)) & 1u;
    }
    return left ? f.left_child[g] : f.right_child[g];
  }
  if (isnan(fval) && mt != 2) fval = 0.0;
  if ((mt == 1 && fabs(fval) <= 1e-35) || (mt == 2 && isnan(fval))) left = (dt & 2) != 0;
  else left = fval <= f.threshold[g];
  return left ? f.left_child[g] : f.right_child[g];
}
template <typename T>
__device__ __forceinline__ int d_tree_leaf(const ForestDev& f, int t, const T* __restrict__ row) {
  if (f.num_leaves[t] <= 1) return 0;
  const int nb = f.tree_offset[t];
  int node = 0;
  while (node >= 0) node = d_node_child(f, nb + node, row);
  return ~node;
}
template <typename T>
__global__ void __launch_bounds__(256)
k_predict_raw(ForestDev f, const T* __restrict__ X, long long nrow, int ncol, int K, int t0, int t1, double* __restrict__ out) {
  const long long total = nrow * K;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = e / K;
    const int k = static_cast<int>(e - r * K);
    const T* row = X + r * ncol;
    double acc = 0.0;
    for (int t = t0 + k; t < t1; t += K) acc += f.leaf_value[f.leaf_offset[t] + d_tree_leaf(f, t, row)];
    out[e] = acc;
  }
}
template <typename T>
__global__ void __launch_bounds__(256)
k_predict_leaf(ForestDev f, const T* __restrict__ X, long long nrow, int ncol, int t0, int t1, double* __restrict__ out) {
  const int nt = t1 - t0;
  const long long total = nrow * nt;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = e / nt;
    const int t = t0 + static_cast<int>(e - r * nt);
    out[e] = static_cast<double>(d_tree_leaf(f, t, X + r * ncol));
  }
}

// ---------------------------------------------------------------- batched TreeSHAP (C_API_PREDICT_CONTRIB)
// One thread per row walks every tree of the model in model order with the path-dependent TreeSHAP recursion of Lundberg et al.
// (the algorithm behind [UPSTREAM] Tree::PredictContrib), turned into an explicit stack: a frame = (node, unique depth, parent
// path offset, zero/one fractions, feature).  The hot child is expanded before the cold one, children write their paths
// behind the parent's, so the parent's path is still intact when the cold frame is popped.  Same fp64 operation order as the host
// predictor (HostTree::ShapRecurse) => identical contributions.  Scratch per thread: path_stride PathElem + frame_stride frames.
struct ShapPathElem { int feature; int pad; double zf, of, pw; };
struct ShapFrame { int node, depth, parent_off, feature; double pzf, pof; };

__device__ __forceinline__ void d_shap_extend(ShapPathElem* p, int depth, double zf, double of, int fi) {
  p[depth].feature = fi; p[depth].zf = zf; p[depth].of = of; p[depth].pw = depth == 0 ? 1.0 : 0.0;
  for (int i = depth - 1; i >= 0; --i) {
    p[i + 1].pw += of * p[i].pw * (i + 1) / static_cast<double>(depth + 1);
    p[i].pw = zf * p[i].pw * (depth - i) / static_cast<double>(depth + 1);
  }
}
__device__ __forceinline__ void d_shap_unwind(ShapPathElem* p, int depth, int pi) {
  const double of = p[pi].of, zf = p[pi].zf;
  double next = p[depth].pw;
  for (int i = depth - 1; i >= 0; --i) {
    if (of != 0) {
      const double tmp = p[i].pw;
      p[i].pw = next * (depth + 1) / static_cast<double>((i + 1) * of);
      next = tmp - p[i].pw * zf * (depth - i) / static_cast<double>(depth + 1);
    } else {
      p[i].pw = (p[i].pw * (depth + 1)) / static_cast<double>(zf * (depth - i));
    }
  }
  for (int i = pi; i < depth; ++i) { p[i].feature = p[i + 1].feature; p[i].zf = p[i + 1].zf; p[i].of = p[i + 1].of; }
}
__device__ __forceinline__ double d_shap_unwound_sum(const ShapPathElem* p, int depth, int pi) {
  const double of = p[pi].of, zf = p[pi].zf;
  double next = p[depth].pw, total = 0;
  for (int i = depth - 1; i >= 0; --i) {
    if (of != 0) {
      const double tmp = next * (depth + 1) / static_cast<double>((i + 1) * of);
      total += tmp;
      next = p[i].pw - tmp * zf * ((depth - i) / static_cast<double>(depth + 1));
    } else {
      total += (p[i].pw / zf) / ((depth - i) / static_cast<double>(depth + 1));
    }
  }
  return total;
}
template <typename T>
__global__ void __launch_bounds__(128)
k_predict_contrib(ForestDev f, const T* __restrict__ X, long long nrow, int ncol, int K, int t0, int t1, int F1, ShapPathElem* __restrict__ path_scratch,
                  int path_stride, ShapFrame* __restrict__ frame_scratch, int frame_stride, double* __restrict__ out) {
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  ShapPathElem* const base = path_scratch + tid * path_stride;
  ShapFrame* const stack = frame_scratch + tid * frame_stride;
  for (long long r = tid; r < nrow; r += static_cast<long long>(gridDim.x) * blockDim.x) {
    const T* row = X + r * ncol;
    for (int t = t0; t < t1; ++t) {
      double* phi = out + (r * K + (t % K)) * F1;
      phi[F1 - 1] += f.expected[t];
      if (f.num_leaves[t] <= 1) continue;
      const int nb = f.tree_offset[t], lb = f.leaf_offset[t];
      int sp = 0;
      stack[sp++] = ShapFrame{0, 0, 0, -1, 1.0, 1.0};
      while (sp > 0) {
        const ShapFrame fr = stack[--sp];
        int depth = fr.depth;
        ShapPathElem* path = base + fr.parent_off + depth;
        const ShapPathElem* parent = base + fr.parent_off;
        for (int i = 0; i < depth; ++i) path[i] = parent[i];
        d_shap_extend(path, depth, fr.pzf, fr.pof, fr.feature);
        if (fr.node < 0) {
          const double lv = f.leaf_value[lb + ~fr.node];
          for (int i = 1; i <= depth; ++i) {
            const double w = d_shap_unwound_sum(path, depth, i);
            phi[path[i].feature] += w * (path[i].of - path[i].zf) * lv;
          }
          continue;
        }
        const int g = nb + fr.node;
        const int hot = d_node_child(f, g, row);
        const int cold = hot == f.left_child[g] ? f.right_child[g] : f.left_child[g];
        const double w = f.node_count[g];
        const double hot_zf = (hot >= 0 ? f.node_count[nb + hot] : f.leaf_count[lb + ~hot]) / w;
        const double cold_zf = (cold >= 0 ? f.node_count[nb + cold] : f.leaf_count[lb + ~cold]) / w;
        double inc_zf = 1, inc_of = 1;
        const int sf = f.split_feature[g];
        int pi = 0;
        for (; pi <= depth; ++pi) if (path[pi].feature == sf) break;
        if (pi != depth + 1) {
          inc_zf = path[pi].zf; inc_of = path[pi].of;
          d_shap_unwind(path, depth, pi);
          depth -= 1;
        }
        const int off = static_cast<int>(path - base);
        stack[sp++] = ShapFrame{cold, depth + 1, off, sf, cold_zf * inc_zf, 0.0};
        stack[sp++] = ShapFrame{hot, depth + 1, off, sf, hot_zf * inc_zf, inc_of};
      }
    }
  }
}

// ---------------------------------------------------------------- batched prediction of CSR rows
// The predict kernels above read a CSR row through a dense [rows][U] row of "slots": one per distinct split feature of the trees
// walked, with the forest's split_feature remapped to slots.  One warp per row zero-fills its slots, then stores the row's entries
// 32 at a time in CSR order.  Values match LGBM_BoosterPredictForCSRSingle's densified row: a missing entry is 0, stored zeros and
// NaN are kept, an index outside [0, num_feature) or of a feature no tree splits on is dropped, and of repeated indices the last
// wins: within a stride the highest lane of each slot stores, and __syncwarp orders the strides.
__global__ void __launch_bounds__(256)
k_csr_to_slots(const long long* __restrict__ indptr, const int* __restrict__ indices, const double* __restrict__ data, long long nrow,
               const int* __restrict__ slot_of_feature, int num_feature, int U, double* __restrict__ X) {
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long r = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5; r < nrow; r += warps) {
    double* row = X + r * U;
    for (int s = lane; s < U; s += 32) row[s] = 0.0;
    __syncwarp();
    const long long b = indptr[r + 1];
    for (long long k0 = indptr[r]; k0 < b; k0 += 32) {
      const long long k = k0 + lane;
      int slot = -1;
      double v = 0.0;
      if (k < b) {
        const int j = indices[k];
        if (j >= 0 && j < num_feature) { slot = slot_of_feature[j]; v = data[k]; }
      }
      const unsigned same = __match_any_sync(0xffffffffu, slot);
      if (slot >= 0 && lane == 31 - __clz(same)) row[slot] = v;
      __syncwarp();
    }
  }
}
// contributions per slot [rows][K][U+1] (expected value last) -> LightGBM's dense layout [rows][K][F1] in a zero-filled `out`
__global__ void k_contrib_slots_to_features(const double* __restrict__ in, long long rows_k, int U, const int* __restrict__ feature_of_slot,
                                            int F1, double* __restrict__ out) {
  const long long total = rows_k * (U + 1);
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long rk = e / (U + 1);
    const int s = static_cast<int>(e - rk * (U + 1));
    out[rk * F1 + (s == U ? F1 - 1 : feature_of_slot[s])] = in[e];
  }
}

}  // namespace b200gbm
