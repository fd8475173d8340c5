// Host-side bin finder: value -> bin boundaries for one feature.
//
// Replaces [UPSTREAM lightgbmlib 3.2.110] BinMapper::FindBin / GreedyFindBin / FindBinWithZeroAsOneBin,
// which the reference reaches through LGBM_DatasetCreateFromMat
// (lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/dataset/DatasetAggregator.scala:335-343)
// with the dataset parameters of LightGBMBase.scala:265-272.  Semantics: SURVEY.md Appendix A.2.
// The boundaries are found on the host from a <=200 000-row sample (one-off, O(sample*F log)); the
// N x F value->bin mapping itself is the CUDA kernel k_bin_rows (kernels.cuh).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <limits>
#include <map>
#include <set>
#include <string>
#include <vector>

namespace b200gbm {

constexpr double kEps = 1e-15;
constexpr double kZeroThr = 1e-35;
constexpr double kSparseThr = 0.7;
enum : int { MISSING_NONE = 0, MISSING_ZERO = 1, MISSING_NAN = 2 };

// LightGBM's LCG (utils/random.h); Sample() picks the rows that define the bins.
class LcgRandom {
 public:
  explicit LcgRandom(int seed) : x_(static_cast<unsigned>(seed)) {}
  std::vector<int> Sample(int n, int k) {
    std::vector<int> out;
    if (k > n || k <= 0) return out;
    out.reserve(k);
    if (k == n) {
      for (int i = 0; i < n; ++i) out.push_back(i);
    } else if (k > 1 && k > (n / std::log2(static_cast<double>(k)))) {
      for (int i = 0; i < n; ++i) {
        double prob = (k - static_cast<double>(out.size())) / static_cast<double>(n - i);
        if (NextFloat() < prob) out.push_back(i);
      }
    } else {
      std::set<int> chosen;
      for (int r = n - k; r < n; ++r) {
        int v = static_cast<int>(Next31() % static_cast<unsigned>(r));
        if (!chosen.insert(v).second) chosen.insert(r);
      }
      out.assign(chosen.begin(), chosen.end());
    }
    return out;
  }
  float NextFloat() { return static_cast<float>((Step() >> 16) & 0x7FFF) / 32768.0f; }
  // the stream position, so that the device can continue the stream within a tree (TreeLearner, per-node sampling)
  unsigned state() const { return x_; }
  void set_state(unsigned x) { x_ = x; }

 private:
  unsigned Step() { x_ = 214013u * x_ + 2531011u; return x_; }
  unsigned Next31() { return Step() & 0x7FFFFFFFu; }
  unsigned x_;
};

struct FeatureBins {
  int num_bin = 1;
  int missing_type = MISSING_NONE;
  bool trivial = true;
  bool categorical = false;
  std::vector<int> bin_to_cat;      // categorical: bin -> category value; bin 0 = -1 (NaN, negative, rare or unseen categories)
  std::vector<int> sorted_cats;     // categories in ascending order ...
  std::vector<int> sorted_bins;     // ... and the bin of each (device lookup table = binary search over sorted_cats)
  uint32_t default_bin = 0;
  uint32_t most_freq_bin = 0;
  double sparse_rate = 1.0;
  double min_val = 0, max_val = 0;
  std::vector<double> upper;   // upper[b] = inclusive upper bound of bin b; NaN bin (if any) is last

  uint32_t ValueToBin(double v) const {
    if (categorical) {
      if (std::isnan(v)) return 0;
      const int iv = static_cast<int>(v);
      if (iv < 0) return 0;
      auto it = std::lower_bound(sorted_cats.begin(), sorted_cats.end(), iv);
      return (it != sorted_cats.end() && *it == iv) ? static_cast<uint32_t>(sorted_bins[it - sorted_cats.begin()]) : 0u;
    }
    if (std::isnan(v)) {
      if (missing_type == MISSING_NAN) return static_cast<uint32_t>(num_bin - 1);
      v = 0.0;
    }
    int lo = 0, hi = num_bin - 1 - (missing_type == MISSING_NAN ? 1 : 0);
    while (lo < hi) {
      int mid = (hi + lo - 1) / 2;
      if (v <= upper[mid]) hi = mid; else lo = mid + 1;
    }
    return static_cast<uint32_t>(lo);
  }
  std::string InfoString() const {
    if (trivial) return "none";
    if (categorical) {
      std::string r;
      for (size_t i = 0; i < bin_to_cat.size(); ++i) r += (i ? ":" : "") + std::to_string(bin_to_cat[i]);
      return r;
    }
    char buf[96];
    snprintf(buf, sizeof(buf), "[%.17g:%.17g]", min_val, max_val);
    return buf;
  }
};

namespace binfind {

inline double NextUp(double a) { return std::nextafter(a, std::numeric_limits<double>::infinity()); }
inline bool SameOrAdjacent(double a, double b) { return b <= NextUp(a); }   // CheckDoubleEqualOrdered

struct Distinct {
  std::vector<double> val;
  std::vector<int> cnt;
  void Push(double v, int c) { val.push_back(v); cnt.push_back(c); }
};

// equal-frequency placement with "big count" values isolated  (GreedyFindBin)
inline std::vector<double> Greedy(const double* v, const int* c, int nd, int max_bin, int total, int min_in_bin) {
  const double inf = std::numeric_limits<double>::infinity();
  std::vector<double> bounds;
  if (nd <= max_bin) {
    int acc = 0;
    for (int i = 0; i + 1 < nd; ++i) {
      acc += c[i];
      if (acc < min_in_bin) continue;
      double mid = NextUp((v[i] + v[i + 1]) / 2.0);
      if (bounds.empty() || !SameOrAdjacent(bounds.back(), mid)) { bounds.push_back(mid); acc = 0; }
    }
    bounds.push_back(inf);
    return bounds;
  }
  if (min_in_bin > 0) max_bin = std::max(1, std::min(max_bin, total / min_in_bin));
  double mean_size = static_cast<double>(total) / max_bin;
  int bins_left = max_bin, samples_left = total;
  std::vector<char> heavy(nd, 0);
  for (int i = 0; i < nd; ++i)
    if (c[i] >= mean_size) { heavy[i] = 1; --bins_left; samples_left -= c[i]; }
  mean_size = static_cast<double>(samples_left) / bins_left;
  std::vector<double> hi_of(max_bin, inf), lo_of(max_bin, inf);
  int nb = 0, acc = 0;
  lo_of[0] = v[0];
  for (int i = 0; i + 1 < nd; ++i) {
    if (!heavy[i]) samples_left -= c[i];
    acc += c[i];
    bool close = heavy[i] || acc >= mean_size || (heavy[i + 1] && acc >= std::max(1.0, mean_size * 0.5f));
    if (!close) continue;
    hi_of[nb] = v[i];
    ++nb;
    lo_of[nb] = v[i + 1];
    if (nb >= max_bin - 1) break;
    acc = 0;
    if (!heavy[i]) { --bins_left; mean_size = samples_left / static_cast<double>(bins_left); }
  }
  ++nb;
  for (int i = 0; i + 1 < nb; ++i) {
    double mid = NextUp((hi_of[i] + lo_of[i + 1]) / 2.0);
    if (bounds.empty() || !SameOrAdjacent(bounds.back(), mid)) bounds.push_back(mid);
  }
  bounds.push_back(inf);
  return bounds;
}

// zero always gets its own bin (-1e-35, 1e-35]; negative / positive sides binned separately
inline std::vector<double> ZeroAsOneBin(const Distinct& d, int max_bin, int total, int min_in_bin) {
  const int nd = static_cast<int>(d.val.size());
  int n_neg = 0, n_pos = 0, n_zero = 0, first_nonneg = nd;
  for (int i = 0; i < nd; ++i) {
    if (d.val[i] <= -kZeroThr) n_neg += d.cnt[i];
    else if (d.val[i] > kZeroThr) n_pos += d.cnt[i];
    else n_zero += d.cnt[i];
  }
  for (int i = 0; i < nd; ++i) if (d.val[i] > -kZeroThr) { first_nonneg = i; break; }
  std::vector<double> bounds;
  if (first_nonneg > 0 && max_bin > 1) {
    int budget = static_cast<int>(static_cast<double>(n_neg) / (total - n_zero) * (max_bin - 1));
    budget = std::max(1, budget);
    bounds = Greedy(d.val.data(), d.cnt.data(), first_nonneg, budget, n_neg, min_in_bin);
    if (!bounds.empty()) bounds.back() = -kZeroThr;
  }
  int first_pos = -1;
  for (int i = first_nonneg; i < nd; ++i) if (d.val[i] > kZeroThr) { first_pos = i; break; }
  int right_budget = max_bin - 1 - static_cast<int>(bounds.size());
  if (first_pos >= 0 && right_budget > 0) {
    std::vector<double> rb = Greedy(d.val.data() + first_pos, d.cnt.data() + first_pos, nd - first_pos, right_budget, n_pos, min_in_bin);
    bounds.push_back(kZeroThr);
    bounds.insert(bounds.end(), rb.begin(), rb.end());
  } else {
    bounds.push_back(std::numeric_limits<double>::infinity());
  }
  return bounds;
}

}  // namespace binfind

// Categorical feature: integer categories ranked by sample count; bin 0 is the catch-all (NaN / negative / rare / unseen),
// categories are kept until 99 % of the non-missing mass is covered and at least min(#distinct, max_bin) bins exist
// ([UPSTREAM] BinMapper::FindBin, CategoricalBin branch; SURVEY.md A.2).
inline FeatureBins FindCategoricalBins(std::vector<double>* nonzero, int total_sample, int max_bin, int min_data_in_bin, int filter_cnt,
                                       bool pre_filter) {
  FeatureBins fb;
  fb.categorical = true;
  std::vector<double>& v = *nonzero;
  int n_nan = 0;
  std::map<int, int> count_of;     // category -> samples (ascending by category)
  for (double x : v) {
    if (std::isnan(x)) { ++n_nan; continue; }
    const int c = static_cast<int>(x);
    if (c < 0) ++n_nan; else ++count_of[c];
  }
  const int n_zero = total_sample - static_cast<int>(v.size());
  if (n_zero > 0) count_of[0] += n_zero;            // the implied zeros are category 0
  struct CC { int cat, cnt; };
  std::vector<CC> ranked;
  for (auto& kv : count_of) ranked.push_back({kv.first, kv.second});
  std::stable_sort(ranked.begin(), ranked.end(), [](const CC& a, const CC& b) { return a.cnt > b.cnt; });
  fb.num_bin = 1;
  fb.bin_to_cat.assign(1, -1);
  std::vector<int> in_bin(1, 0);
  const int rest = total_sample - n_nan;
  if (rest > 0) {
    const int cut = static_cast<int>(rest * 0.99f + 0.5);
    int distinct = static_cast<int>(ranked.size()) + (n_nan > 0 ? 1 : 0);
    const int want_bins = std::min(distinct, max_bin);
    int used = 0;
    size_t k = 0;
    while (k < ranked.size() && (used < cut || fb.num_bin < want_bins)) {
      if (ranked[k].cnt < min_data_in_bin && k > 1) break;
      fb.bin_to_cat.push_back(ranked[k].cat);
      in_bin.push_back(ranked[k].cnt);
      used += ranked[k].cnt;
      ++fb.num_bin; ++k;
    }
    fb.missing_type = (k == ranked.size() && n_nan == 0) ? MISSING_NONE : MISSING_NAN;
    in_bin[0] = total_sample - used;
  }
  std::vector<std::pair<int, int>> byc;
  for (int b = 1; b < fb.num_bin; ++b) byc.emplace_back(fb.bin_to_cat[b], b);
  std::sort(byc.begin(), byc.end());
  for (auto& p : byc) { fb.sorted_cats.push_back(p.first); fb.sorted_bins.push_back(p.second); }
  fb.min_val = byc.empty() ? 0 : byc.front().first;
  fb.max_val = byc.empty() ? 0 : byc.back().first;
  fb.trivial = fb.num_bin <= 1;
  if (!fb.trivial && pre_filter && in_bin.size() <= 2) {
    bool ok = false;
    for (size_t b = 0; b + 1 < in_bin.size(); ++b) ok |= in_bin[b] >= filter_cnt && total_sample - in_bin[b] >= filter_cnt;
    if (!ok) fb.trivial = true;
  }
  if (!fb.trivial) {
    fb.default_bin = fb.ValueToBin(0.0);
    fb.most_freq_bin = static_cast<uint32_t>(std::max_element(in_bin.begin(), in_bin.end()) - in_bin.begin());
    double rate = static_cast<double>(in_bin[fb.most_freq_bin]) / total_sample;
    if (fb.most_freq_bin != fb.default_bin && rate < kSparseThr) fb.most_freq_bin = fb.default_bin;
    fb.sparse_rate = static_cast<double>(in_bin[fb.most_freq_bin]) / total_sample;
  }
  return fb;
}

// nonzero: sampled values with |v| > 1e-35 or NaN (consumed); total_sample: rows sampled (zeros implied)
inline FeatureBins FindFeatureBins(std::vector<double>* nonzero, int total_sample, int max_bin, int min_data_in_bin,
                                   int filter_cnt, bool pre_filter, bool use_missing, bool zero_as_missing) {
  FeatureBins fb;
  std::vector<double>& v = *nonzero;
  const int given = static_cast<int>(v.size());
  v.erase(std::remove_if(v.begin(), v.end(), [](double x) { return std::isnan(x); }), v.end());
  const int m = static_cast<int>(v.size());
  int n_nan = 0;
  if (!use_missing) fb.missing_type = MISSING_NONE;
  else if (zero_as_missing) fb.missing_type = MISSING_ZERO;
  else if (m == given) fb.missing_type = MISSING_NONE;
  else { fb.missing_type = MISSING_NAN; n_nan = given - m; }
  const int n_zero = total_sample - m - n_nan;
  std::stable_sort(v.begin(), v.end());

  binfind::Distinct d;
  if (m == 0 || (v[0] > 0.0 && n_zero > 0)) d.Push(0.0, n_zero);
  if (m > 0) d.Push(v[0], 1);
  for (int i = 1; i < m; ++i) {
    if (binfind::SameOrAdjacent(v[i - 1], v[i])) { d.val.back() = v[i]; ++d.cnt.back(); continue; }
    if (v[i - 1] < 0.0 && v[i] > 0.0) d.Push(0.0, n_zero);
    d.Push(v[i], 1);
  }
  if (m > 0 && v[m - 1] < 0.0 && n_zero > 0) d.Push(0.0, n_zero);
  fb.min_val = d.val.front();
  fb.max_val = d.val.back();

  if (fb.missing_type == MISSING_NAN) {
    fb.upper = binfind::ZeroAsOneBin(d, max_bin - 1, total_sample - n_nan, min_data_in_bin);
    fb.upper.push_back(std::numeric_limits<double>::quiet_NaN());
  } else {
    fb.upper = binfind::ZeroAsOneBin(d, max_bin, total_sample, min_data_in_bin);
    if (fb.missing_type == MISSING_ZERO && fb.upper.size() == 2) fb.missing_type = MISSING_NONE;
  }
  fb.num_bin = static_cast<int>(fb.upper.size());

  std::vector<int> in_bin(fb.num_bin, 0);
  for (size_t i = 0, b = 0; i < d.val.size(); ++i) {
    while (d.val[i] > fb.upper[b] && static_cast<int>(b) < fb.num_bin - 1) ++b;
    in_bin[b] += d.cnt[i];
  }
  if (fb.missing_type == MISSING_NAN) in_bin[fb.num_bin - 1] = n_nan;

  fb.trivial = fb.num_bin <= 1;
  if (!fb.trivial && pre_filter) {
    // no threshold can leave filter_cnt samples on both sides => feature can never split
    bool can_split = false;
    int left = 0;
    for (int b = 0; b + 1 < fb.num_bin && !can_split; ++b) {
      left += in_bin[b];
      can_split = left >= filter_cnt && total_sample - left >= filter_cnt;
    }
    if (!can_split) fb.trivial = true;
  }
  if (!fb.trivial) {
    fb.default_bin = fb.ValueToBin(0.0);
    fb.most_freq_bin = static_cast<uint32_t>(std::max_element(in_bin.begin(), in_bin.end()) - in_bin.begin());
    double rate = static_cast<double>(in_bin[fb.most_freq_bin]) / total_sample;
    if (fb.most_freq_bin != fb.default_bin && rate < kSparseThr) fb.most_freq_bin = fb.default_bin;
    fb.sparse_rate = static_cast<double>(in_bin[fb.most_freq_bin]) / total_sample;
  }
  return fb;
}

}  // namespace b200gbm
