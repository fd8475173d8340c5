// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load this library.
//
// CPU restatement (C++17 + OpenMP) of the LightGBM-on-Spark training hot path that MMLSpark
// reaches through SWIG (SURVEY.md §8a): bin finding + binning, objectives, per-leaf fp64
// feature histograms, numerical and categorical best-split scans, leaf-wise growth with histogram
// subtraction, bagging / GOSS / RF / DART, leaf-output renewal, GBDT loop and model-text v3 writer.
//
// PARITY UNPINNED: the arithmetic lives in the un-vendored Maven artifact
// com.microsoft.ml.lightgbm:lightgbmlib:3.2.110 (reference build.sbt:222), whose source
// is not part of the reference.  Everything here restates the published
// LightGBM v3.2.x algorithm from knowledge and is anchored on the reference's call sites:
//   dataset creation   lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/dataset/DatasetAggregator.scala:331-352
//   dataset params     lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/LightGBMBase.scala:265-272
//   booster params     lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/params/TrainParams.scala:47-63
//   one iteration      lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/booster/LightGBMBooster.scala:351-361
//   training loop      lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/TrainUtils.scala:92-159
//   model string       lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/booster/LightGBMBooster.scala:269-274
// The reference's own tests hold no bit-level vectors for this path (SURVEY.md §8c); its only
// known-answer tests (countCardinality, VerifyLightGBMRanker.scala:127-137) are checked in tests/.
// Independent cross-check (tests/test_oracle_vs_sklearn_cpu.py): on data where the bin finders agree by
// construction this oracle and scikit-learn's HistGradientBoosting (a separate implementation of the same
// algorithm family) fit the same model to 1e-13 — regression, binary, max_depth, NaN default direction,
// weights, categorical splits — once LightGBM's is_splittable inheritance rule is accounted for.  That
// pins the shared algorithm, not LightGBM's remaining idiosyncrasies (bin finder, tie-breaks, DART/GOSS
// details), which stay unpinned against the real binary.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <numeric>
#include <set>
#include <sstream>
#include <string>
#include <vector>
#include <functional>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace orc {

constexpr double kEpsilon = 1e-15;
constexpr double kZeroThreshold = 1e-35;
constexpr double kMinScore = -std::numeric_limits<double>::infinity();
constexpr double kSparseThreshold = 0.7;

// ------------------------------------------------------------------ config
// Grammar: space separated key=value, empty values allowed ("metric="), later keys win
// (TrainParams.scala:47-63 emits `metric=` twice for classifiers).
struct Config {
  std::string objective = "regression";
  std::string boosting = "gbdt";
  std::string metric;
  int num_iterations = 100;
  double learning_rate = 0.1;
  int num_leaves = 31;
  int max_bin = 255;
  int min_data_in_leaf = 20;
  double min_sum_hessian_in_leaf = 1e-3;
  double lambda_l1 = 0, lambda_l2 = 0, min_gain_to_split = 0, max_delta_step = 0;
  int max_depth = -1;
  int num_class = 1;
  bool is_unbalance = false;
  double scale_pos_weight = 1.0;
  bool boost_from_average = true;
  double sigmoid = 1.0;
  int bin_construct_sample_cnt = 200000;
  int min_data_in_bin = 3;
  int data_random_seed = 1;
  bool use_missing = true, zero_as_missing = false, feature_pre_filter = true;
  int lambdarank_truncation_level = 30;
  bool lambdarank_norm = true;
  std::vector<double> label_gain;
  std::vector<int> eval_at;
  std::vector<int> categorical_feature;
  int num_machines = 1;
  double feature_fraction = 1.0;
  int feature_fraction_seed = 2;
  double alpha = 0.9, fair_c = 1.0, poisson_max_delta_step = 0.7, tweedie_variance_power = 1.5;
  int max_cat_threshold = 32, max_cat_to_onehot = 4, min_data_per_group = 100;
  double cat_l2 = 10.0, cat_smooth = 10.0;
  double bagging_fraction = 1.0, pos_bagging_fraction = 1.0, neg_bagging_fraction = 1.0, top_rate = 0.2, other_rate = 0.1;
  int bagging_freq = 0, bagging_seed = 3;
  double drop_rate = 0.1, skip_drop = 0.5;
  int max_drop = 50, drop_seed = 4;
  bool uniform_drop = false, xgboost_dart_mode = false;
  bool oracle_inherit_splittable = true;   // test-only switch: false = children re-examine every feature (what sklearn's HGB does)
  std::string tree_learner = "serial";
  int verbosity = 1;
  std::map<std::string, std::string> raw;

  static bool to_bool(const std::string& v) {
    return v == "true" || v == "True" || v == "TRUE" || v == "1" || v == "+";
  }
  static std::string canon(const std::string& k) {
    static const std::map<std::string, std::string> alias = {
        {"boosting_type", "boosting"}, {"boost", "boosting"}, {"application", "objective"},
        {"app", "objective"}, {"objective_type", "objective"}, {"num_iteration", "num_iterations"},
        {"num_trees", "num_iterations"}, {"num_round", "num_iterations"}, {"n_estimators", "num_iterations"},
        {"shrinkage_rate", "learning_rate"}, {"eta", "learning_rate"}, {"num_leaf", "num_leaves"},
        {"max_leaves", "num_leaves"}, {"min_data_per_leaf", "min_data_in_leaf"}, {"min_data", "min_data_in_leaf"},
        {"min_child_samples", "min_data_in_leaf"}, {"min_sum_hessian_per_leaf", "min_sum_hessian_in_leaf"},
        {"min_sum_hessian", "min_sum_hessian_in_leaf"}, {"min_hessian", "min_sum_hessian_in_leaf"},
        {"min_child_weight", "min_sum_hessian_in_leaf"}, {"reg_alpha", "lambda_l1"}, {"reg_lambda", "lambda_l2"},
        {"lambda", "lambda_l2"}, {"min_split_gain", "min_gain_to_split"}, {"max_position", "lambdarank_truncation_level"},
        {"unbalance", "is_unbalance"}, {"unbalanced_sets", "is_unbalance"}, {"metrics", "metric"},
        {"metric_types", "metric"}, {"subsample_for_bin", "bin_construct_sample_cnt"},
        {"is_pre_partition", "pre_partition"}, {"tree", "tree_learner"}, {"tree_type", "tree_learner"},
        {"tree_learner_type", "tree_learner"}, {"num_classes", "num_class"}, {"ndcg_eval_at", "eval_at"},
        {"ndcg_at", "eval_at"}, {"cat_feature", "categorical_feature"}, {"categorical_column", "categorical_feature"},
        {"num_machine", "num_machines"}, {"verbose", "verbosity"}, {"sub_feature", "feature_fraction"},
        {"colsample_bytree", "feature_fraction"}, {"max_delta", "max_delta_step"}};
    auto it = alias.find(k);
    return it == alias.end() ? k : it->second;
  }
  static std::string canon_objective(const std::string& o) {
    if (o == "regression" || o == "regression_l2" || o == "l2" || o == "mean_squared_error" || o == "mse" ||
        o == "l2_root" || o == "root_mean_squared_error" || o == "rmse")
      return "regression";
    if (o == "softmax") return "multiclass";
    if (o == "multiclass_ova" || o == "ova" || o == "ovr") return "multiclassova";
    if (o == "xentropy") return "cross_entropy";
    if (o == "l1" || o == "mean_absolute_error" || o == "mae") return "regression_l1";
    if (o == "mean_absolute_percentage_error") return "mape";
    return o;
  }
  void parse(const char* s) {
    if (!s) return;
    std::istringstream is(s);
    std::string tok;
    while (is >> tok) {
      auto p = tok.find('=');
      if (p == std::string::npos) continue;
      std::string k = canon(tok.substr(0, p)), v = tok.substr(p + 1);
      raw[k] = v;
    }
    auto geti = [&](const char* k, int& d) { auto it = raw.find(k); if (it != raw.end() && !it->second.empty()) d = std::atoi(it->second.c_str()); };
    auto getd = [&](const char* k, double& d) { auto it = raw.find(k); if (it != raw.end() && !it->second.empty()) d = std::atof(it->second.c_str()); };
    auto getb = [&](const char* k, bool& d) { auto it = raw.find(k); if (it != raw.end() && !it->second.empty()) d = to_bool(it->second); };
    auto gets = [&](const char* k, std::string& d) { auto it = raw.find(k); if (it != raw.end()) d = it->second; };
    gets("objective", objective); objective = canon_objective(objective);
    gets("boosting", boosting); gets("metric", metric); gets("tree_learner", tree_learner);
    geti("num_iterations", num_iterations); getd("learning_rate", learning_rate); geti("num_leaves", num_leaves);
    geti("max_bin", max_bin); geti("min_data_in_leaf", min_data_in_leaf);
    getd("min_sum_hessian_in_leaf", min_sum_hessian_in_leaf); getd("lambda_l1", lambda_l1);
    getd("lambda_l2", lambda_l2); getd("min_gain_to_split", min_gain_to_split); getd("max_delta_step", max_delta_step);
    geti("max_depth", max_depth); geti("num_class", num_class); getb("is_unbalance", is_unbalance);
    getd("scale_pos_weight", scale_pos_weight); getb("boost_from_average", boost_from_average);
    getd("sigmoid", sigmoid); geti("bin_construct_sample_cnt", bin_construct_sample_cnt);
    geti("min_data_in_bin", min_data_in_bin); geti("data_random_seed", data_random_seed);
    getb("use_missing", use_missing); getb("zero_as_missing", zero_as_missing);
    getb("feature_pre_filter", feature_pre_filter); geti("lambdarank_truncation_level", lambdarank_truncation_level);
    getb("lambdarank_norm", lambdarank_norm); geti("num_machines", num_machines);
    getd("feature_fraction", feature_fraction); geti("verbosity", verbosity); geti("feature_fraction_seed", feature_fraction_seed);
    getd("alpha", alpha); getd("fair_c", fair_c); getd("poisson_max_delta_step", poisson_max_delta_step);
    getd("tweedie_variance_power", tweedie_variance_power);
    geti("max_cat_threshold", max_cat_threshold); geti("max_cat_to_onehot", max_cat_to_onehot); geti("min_data_per_group", min_data_per_group);
    getd("cat_l2", cat_l2); getd("cat_smooth", cat_smooth);
    getd("pos_bagging_fraction", pos_bagging_fraction); getd("neg_bagging_fraction", neg_bagging_fraction);
    getd("bagging_fraction", bagging_fraction); geti("bagging_freq", bagging_freq); geti("bagging_seed", bagging_seed);
    getd("top_rate", top_rate); getd("other_rate", other_rate);
    getd("drop_rate", drop_rate); getd("skip_drop", skip_drop); geti("max_drop", max_drop); geti("drop_seed", drop_seed);
    getb("uniform_drop", uniform_drop); getb("xgboost_dart_mode", xgboost_dart_mode);
    getb("oracle_inherit_splittable", oracle_inherit_splittable);
    if (boosting == "random_forest") boosting = "rf";
    if (boosting == "gbrt") boosting = "gbdt";
    auto split_list = [&](const char* k, auto& out, auto conv) {
      auto it = raw.find(k);
      if (it == raw.end() || it->second.empty()) return;
      out.clear();
      std::stringstream ss(it->second);
      std::string x;
      while (std::getline(ss, x, ',')) if (!x.empty()) out.push_back(conv(x));
    };
    split_list("label_gain", label_gain, [](const std::string& x) { return std::atof(x.c_str()); });
    split_list("eval_at", eval_at, [](const std::string& x) { return std::atoi(x.c_str()); });
    split_list("categorical_feature", categorical_feature, [](const std::string& x) { return std::atoi(x.c_str()); });
  }
};

// ------------------------------------------------------------------ LCG  [UPSTREAM utils/random.h]
struct Random {
  unsigned int x = 123456789;
  explicit Random(int seed) : x(static_cast<unsigned>(seed)) {}
  int RandInt16() { x = 214013u * x + 2531011u; return static_cast<int>((x >> 16) & 0x7FFF); }
  int RandInt32() { x = 214013u * x + 2531011u; return static_cast<int>(x & 0x7FFFFFFF); }
  int NextInt(int lo, int hi) { return RandInt32() % (hi - lo) + lo; }
  float NextFloat() { return static_cast<float>(RandInt16()) / 32768.0f; }
  std::vector<int> Sample(int N, int K) {
    std::vector<int> ret;
    ret.reserve(K > 0 ? K : 0);
    if (K > N || K <= 0) return ret;
    if (K == N) { for (int i = 0; i < N; ++i) ret.push_back(i); return ret; }
    if (K > 1 && K > (N / std::log2(static_cast<double>(K)))) {
      for (int i = 0; i < N; ++i) {
        double prob = (K - static_cast<double>(ret.size())) / static_cast<double>(N - i);
        if (NextFloat() < prob) ret.push_back(i);
      }
    } else {
      std::set<int> s;
      for (int r = N - K; r < N; ++r) {
        int v = NextInt(0, r);
        if (!s.insert(v).second) s.insert(r);
      }
      for (int v : s) ret.push_back(v);
    }
    return ret;
  }
};

// ------------------------------------------------------------------ bin mapper [UPSTREAM io/bin.cpp]
enum MissingType { kMissNone = 0, kMissZero = 1, kMissNaN = 2 };

inline bool CheckDoubleEqualOrdered(double a, double b) { return b <= std::nextafter(a, INFINITY); }
inline double GetDoubleUpperBound(double a) { return std::nextafter(a, INFINITY); }

static std::vector<double> GreedyFindBin(const double* dv, const int* cnt, int nd, int max_bin, int total_cnt,
                                         int min_data_in_bin) {
  std::vector<double> ub;
  if (nd <= max_bin) {
    int cur = 0;
    for (int i = 0; i < nd - 1; ++i) {
      cur += cnt[i];
      if (cur >= min_data_in_bin) {
        double val = GetDoubleUpperBound((dv[i] + dv[i + 1]) / 2.0);
        if (ub.empty() || !CheckDoubleEqualOrdered(ub.back(), val)) { ub.push_back(val); cur = 0; }
      }
    }
    ub.push_back(std::numeric_limits<double>::infinity());
  } else {
    if (min_data_in_bin > 0) { max_bin = std::min(max_bin, total_cnt / min_data_in_bin); max_bin = std::max(max_bin, 1); }
    double mean_bin_size = static_cast<double>(total_cnt) / max_bin;
    int rest_bin_cnt = max_bin, rest_sample_cnt = total_cnt;
    std::vector<bool> big(nd, false);
    for (int i = 0; i < nd; ++i)
      if (cnt[i] >= mean_bin_size) { big[i] = true; --rest_bin_cnt; rest_sample_cnt -= cnt[i]; }
    mean_bin_size = static_cast<double>(rest_sample_cnt) / rest_bin_cnt;
    std::vector<double> upper(max_bin, std::numeric_limits<double>::infinity());
    std::vector<double> lower(max_bin, std::numeric_limits<double>::infinity());
    int bin_cnt = 0;
    lower[0] = dv[0];
    int cur = 0;
    for (int i = 0; i < nd - 1; ++i) {
      if (!big[i]) rest_sample_cnt -= cnt[i];
      cur += cnt[i];
      if (big[i] || cur >= mean_bin_size || (big[i + 1] && cur >= std::max(1.0, mean_bin_size * 0.5f))) {
        upper[bin_cnt] = dv[i];
        ++bin_cnt;
        lower[bin_cnt] = dv[i + 1];
        if (bin_cnt >= max_bin - 1) break;
        cur = 0;
        if (!big[i]) { --rest_bin_cnt; mean_bin_size = rest_sample_cnt / static_cast<double>(rest_bin_cnt); }
      }
    }
    ++bin_cnt;
    for (int i = 0; i < bin_cnt - 1; ++i) {
      double val = GetDoubleUpperBound((upper[i] + lower[i + 1]) / 2.0);
      if (ub.empty() || !CheckDoubleEqualOrdered(ub.back(), val)) ub.push_back(val);
    }
    ub.push_back(std::numeric_limits<double>::infinity());
  }
  return ub;
}

static std::vector<double> FindBinWithZeroAsOneBin(const double* dv, const int* cnt, int nd, int max_bin,
                                                   int total_sample_cnt, int min_data_in_bin) {
  std::vector<double> ub;
  int left_cnt_data = 0, cnt_zero = 0, right_cnt_data = 0;
  for (int i = 0; i < nd; ++i) {
    if (dv[i] <= -kZeroThreshold) left_cnt_data += cnt[i];
    else if (dv[i] > kZeroThreshold) right_cnt_data += cnt[i];
    else cnt_zero += cnt[i];
  }
  int left_cnt = -1;
  for (int i = 0; i < nd; ++i) if (dv[i] > -kZeroThreshold) { left_cnt = i; break; }
  if (left_cnt < 0) left_cnt = nd;
  if (left_cnt > 0 && max_bin > 1) {
    int left_max_bin = static_cast<int>(static_cast<double>(left_cnt_data) / (total_sample_cnt - cnt_zero) * (max_bin - 1));
    left_max_bin = std::max(1, left_max_bin);
    ub = GreedyFindBin(dv, cnt, left_cnt, left_max_bin, left_cnt_data, min_data_in_bin);
    if (!ub.empty()) ub.back() = -kZeroThreshold;
  }
  int right_start = -1;
  for (int i = left_cnt; i < nd; ++i) if (dv[i] > kZeroThreshold) { right_start = i; break; }
  int right_max_bin = max_bin - 1 - static_cast<int>(ub.size());
  if (right_start >= 0 && right_max_bin > 0) {
    auto rb = GreedyFindBin(dv + right_start, cnt + right_start, nd - right_start, right_max_bin, right_cnt_data, min_data_in_bin);
    ub.push_back(kZeroThreshold);
    ub.insert(ub.end(), rb.begin(), rb.end());
  } else {
    ub.push_back(std::numeric_limits<double>::infinity());
  }
  return ub;
}

struct BinMapper {
  int num_bin = 1;
  int missing_type = kMissNone;
  bool is_trivial = true;
  bool is_categorical = false;
  double sparse_rate = 1.0;
  std::vector<double> upper;
  std::vector<int> bin_2_cat;            // categorical: bin -> category value (bin 0 = -1: NaN / rare / unseen)
  std::map<int, int> cat_2_bin;
  double min_val = 0, max_val = 0;
  uint32_t default_bin = 0, most_freq_bin = 0;

  uint32_t ValueToBin(double value) const {
    if (is_categorical) {
      if (std::isnan(value)) return 0;
      int iv = static_cast<int>(value);
      if (iv < 0) return 0;
      auto it = cat_2_bin.find(iv);
      return it == cat_2_bin.end() ? 0 : it->second;
    }
    if (std::isnan(value)) {
      if (missing_type == kMissNaN) return num_bin - 1;
      value = 0.0;
    }
    int l = 0, r = num_bin - 1;
    if (missing_type == kMissNaN) r -= 1;
    while (l < r) {
      int m = (r + l - 1) / 2;
      if (value <= upper[m]) r = m; else l = m + 1;
    }
    return l;
  }

  // values: the non-zero (|v|>1e-35 or NaN) sampled values of one feature (modified in place)
  void FindBin(double* values, int num_sample_values, size_t total_sample_cnt, int max_bin, int min_data_in_bin,
               int min_split_data, bool pre_filter, bool use_missing, bool zero_as_missing, bool categorical = false) {
    is_categorical = categorical;
    int na_cnt = 0, tmp = 0;
    for (int i = 0; i < num_sample_values; ++i) if (!std::isnan(values[i])) values[tmp++] = values[i];
    if (!use_missing) missing_type = kMissNone;
    else if (zero_as_missing) missing_type = kMissZero;
    else if (tmp == num_sample_values) missing_type = kMissNone;
    else { missing_type = kMissNaN; na_cnt = num_sample_values - tmp; }
    num_sample_values = tmp;
    default_bin = 0;
    int zero_cnt = static_cast<int>(total_sample_cnt - num_sample_values - na_cnt);
    std::vector<double> dv;
    std::vector<int> counts;
    std::stable_sort(values, values + num_sample_values);
    if (num_sample_values == 0 || (values[0] > 0.0 && zero_cnt > 0)) { dv.push_back(0.0); counts.push_back(zero_cnt); }
    if (num_sample_values > 0) { dv.push_back(values[0]); counts.push_back(1); }
    for (int i = 1; i < num_sample_values; ++i) {
      if (!CheckDoubleEqualOrdered(values[i - 1], values[i])) {
        if (values[i - 1] < 0.0 && values[i] > 0.0) { dv.push_back(0.0); counts.push_back(zero_cnt); }
        dv.push_back(values[i]);
        counts.push_back(1);
      } else {
        dv.back() = values[i];
        ++counts.back();
      }
    }
    if (num_sample_values > 0 && values[num_sample_values - 1] < 0.0 && zero_cnt > 0) { dv.push_back(0.0); counts.push_back(zero_cnt); }
    min_val = dv.front();
    max_val = dv.back();
    int nd = static_cast<int>(dv.size());
    std::vector<int> cnt_in_bin;
    if (categorical) {
      // [UPSTREAM BinMapper::FindBin, CategoricalBin branch] ints; negatives -> NaN; sorted by count; kept until 99 % of the mass
      std::vector<int> dvi, cti;
      for (int i = 0; i < nd; ++i) {
        int val = static_cast<int>(dv[i]);
        if (val < 0) na_cnt += counts[i];
        else if (dvi.empty() || val != dvi.back()) { dvi.push_back(val); cti.push_back(counts[i]); }
        else cti.back() += counts[i];
      }
      num_bin = 1;
      bin_2_cat.assign(1, -1); cat_2_bin.clear(); cat_2_bin[-1] = 0;
      cnt_in_bin.assign(1, 0);
      int rest_cnt = static_cast<int>(total_sample_cnt - na_cnt);
      if (rest_cnt > 0) {
        std::vector<int> order(dvi.size());
        std::iota(order.begin(), order.end(), 0);
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cti[a] > cti[b]; });    // SortForPair(counts, values, 0, true)
        int cut_cnt = RoundIntLocal((total_sample_cnt - na_cnt) * 0.99f);
        int used_cnt = 0;
        int distinct_cnt = static_cast<int>(dvi.size());
        if (na_cnt > 0) ++distinct_cnt;
        int mb = std::min(distinct_cnt, max_bin);
        size_t cur = 0;
        while (cur < order.size() && (used_cnt < cut_cnt || num_bin < mb)) {
          int o = order[cur];
          if (cti[o] < min_data_in_bin && cur > 1) break;
          bin_2_cat.push_back(dvi[o]);
          cat_2_bin[dvi[o]] = num_bin;
          used_cnt += cti[o];
          cnt_in_bin.push_back(cti[o]);
          ++num_bin; ++cur;
        }
        missing_type = (cur == order.size() && na_cnt == 0) ? kMissNone : kMissNaN;
        cnt_in_bin[0] = static_cast<int>(total_sample_cnt - used_cnt);
      }
      is_trivial = num_bin <= 1;
      if (!is_trivial && pre_filter) {
        bool need = true;
        if (cnt_in_bin.size() <= 2) {
          for (size_t i = 0; i + 1 < cnt_in_bin.size(); ++i) {
            int sum_left = cnt_in_bin[i];
            if (sum_left >= min_split_data && static_cast<int>(total_sample_cnt) - sum_left >= min_split_data) { need = false; break; }
          }
        } else need = false;
        if (need) is_trivial = true;
      }
      if (!is_trivial) {
        default_bin = ValueToBin(0);
        most_freq_bin = static_cast<uint32_t>(std::max_element(cnt_in_bin.begin(), cnt_in_bin.end()) - cnt_in_bin.begin());
        double max_sparse_rate = static_cast<double>(cnt_in_bin[most_freq_bin]) / total_sample_cnt;
        if (most_freq_bin != default_bin && max_sparse_rate < kSparseThreshold) most_freq_bin = default_bin;
        sparse_rate = static_cast<double>(cnt_in_bin[most_freq_bin]) / total_sample_cnt;
      } else sparse_rate = 1.0;
      return;
    }
    if (missing_type == kMissZero) {
      upper = FindBinWithZeroAsOneBin(dv.data(), counts.data(), nd, max_bin, static_cast<int>(total_sample_cnt), min_data_in_bin);
      if (upper.size() == 2) missing_type = kMissNone;
    } else if (missing_type == kMissNone) {
      upper = FindBinWithZeroAsOneBin(dv.data(), counts.data(), nd, max_bin, static_cast<int>(total_sample_cnt), min_data_in_bin);
    } else {
      upper = FindBinWithZeroAsOneBin(dv.data(), counts.data(), nd, max_bin - 1, static_cast<int>(total_sample_cnt - na_cnt), min_data_in_bin);
      upper.push_back(std::numeric_limits<double>::quiet_NaN());
    }
    num_bin = static_cast<int>(upper.size());
    cnt_in_bin.assign(num_bin, 0);
    int i_bin = 0;
    for (int i = 0; i < nd; ++i) {
      while (dv[i] > upper[i_bin] && i_bin < num_bin - 1) ++i_bin;
      cnt_in_bin[i_bin] += counts[i];
    }
    if (missing_type == kMissNaN) cnt_in_bin[num_bin - 1] = na_cnt;
    is_trivial = num_bin <= 1;
    if (!is_trivial && pre_filter) {
      // NeedFilter (numerical)
      bool need = true;
      int sum_left = 0;
      for (size_t i = 0; i + 1 < cnt_in_bin.size(); ++i) {
        sum_left += cnt_in_bin[i];
        if (sum_left >= min_split_data && static_cast<int>(total_sample_cnt) - sum_left >= min_split_data) { need = false; break; }
      }
      if (need) is_trivial = true;
    }
    if (!is_trivial) {
      default_bin = ValueToBin(0);
      most_freq_bin = static_cast<uint32_t>(std::max_element(cnt_in_bin.begin(), cnt_in_bin.end()) - cnt_in_bin.begin());
      double max_sparse_rate = static_cast<double>(cnt_in_bin[most_freq_bin]) / total_sample_cnt;
      if (most_freq_bin != default_bin && max_sparse_rate < kSparseThreshold) most_freq_bin = default_bin;
      sparse_rate = static_cast<double>(cnt_in_bin[most_freq_bin]) / total_sample_cnt;
    } else {
      sparse_rate = 1.0;
    }
  }
  static int RoundIntLocal(double x) { return static_cast<int>(x + 0.5); }
  std::string info_string() const {
    if (is_trivial) return "none";
    if (is_categorical) {
      std::string r;
      for (size_t i = 0; i < bin_2_cat.size(); ++i) r += (i ? ":" : "") + std::to_string(bin_2_cat[i]);
      return r;
    }
    char buf[96];
    snprintf(buf, sizeof(buf), "[%.17g:%.17g]", min_val, max_val);
    return buf;
  }
};

// ------------------------------------------------------------------ dataset
struct Dataset {
  int n = 0, F = 0;                       // rows, total features
  Config cfg;                             // dataset-side params
  std::vector<BinMapper> mappers;         // [F]
  std::vector<int> used;                  // inner -> real feature index
  std::vector<int> inner_of;              // real -> inner (-1 if trivial)
  std::vector<uint8_t> bins;              // col-major [n_used][n]  (all features <= 256 bins)
  std::vector<uint16_t> bins16;           // col-major [n_used][n]  (used instead of `bins` when some feature needs more than 256 bins:
                                          //  categorical features are not capped at max_bin — they keep categories until 99 % of the mass)
  bool wide = false;
  inline uint32_t bin_at(size_t u, size_t i) const { return wide ? bins16[u * static_cast<size_t>(n) + i] : bins[u * static_cast<size_t>(n) + i]; }
  void alloc_bins() {
    wide = false;
    for (int f : used) if (mappers[f].num_bin > 256) wide = true;
    if (wide) bins16.resize(used.size() * static_cast<size_t>(n)); else bins.resize(used.size() * static_cast<size_t>(n));
  }
  std::vector<float> label, weight;
  std::vector<double> init_score;
  std::vector<int> query_boundaries;      // ngroup+1
  std::vector<std::string> feature_names;
  std::vector<int> rank_rows;             // emulated data-parallel shards (contiguous row blocks)

  // [UPSTREAM c_api.cpp LGBM_DatasetCreateFromMat + DatasetLoader::ConstructFromSampleData]
  // Multi-rank rule (SURVEY.md fact 9 / A.2): network is up before dataset creation, so rank r finds
  // the bins of the contiguous feature slice [r*step, ...) from ITS OWN local sample.
  void build(const double* X, int nrow, int ncol, const char* params, int num_ranks, const int* rows_per_rank) {
    n = nrow; F = ncol;
    cfg.parse(params);
    rank_rows.assign(rows_per_rank, rows_per_rank + num_ranks);
    mappers.assign(F, BinMapper());
    std::vector<int> start(num_ranks), len(num_ranks);
    int step = (F + num_ranks - 1) / num_ranks;
    if (step < 1) step = 1;
    start[0] = 0;
    for (int i = 0; i < num_ranks - 1; ++i) { len[i] = std::min(step, F - start[i]); start[i + 1] = start[i] + len[i]; }
    len[num_ranks - 1] = F - start[num_ranks - 1];
    int row_off = 0;
    for (int r = 0; r < num_ranks; ++r) {
      int ln = rank_rows[r];
      const double* Xr = X + static_cast<size_t>(row_off) * F;
      Random rnd(cfg.data_random_seed);
      int sample_cnt = ln < cfg.bin_construct_sample_cnt ? ln : cfg.bin_construct_sample_cnt;
      std::vector<int> sidx = rnd.Sample(ln, sample_cnt);
      sample_cnt = static_cast<int>(sidx.size());
      int filter_cnt = static_cast<int>(static_cast<double>(cfg.min_data_in_leaf) * sample_cnt / ln);
      int f0 = num_ranks == 1 ? 0 : start[r], f1 = num_ranks == 1 ? F : start[r] + len[r];
#pragma omp parallel for schedule(dynamic)
      for (int f = f0; f < f1; ++f) {
        std::vector<double> vals;
        vals.reserve(sample_cnt);
        for (int i : sidx) {
          double v = Xr[static_cast<size_t>(i) * F + f];
          if (std::fabs(v) > kZeroThreshold || std::isnan(v)) vals.push_back(v);
        }
        bool is_cat = std::find(cfg.categorical_feature.begin(), cfg.categorical_feature.end(), f) != cfg.categorical_feature.end();
        mappers[f].FindBin(vals.data(), static_cast<int>(vals.size()), sample_cnt, cfg.max_bin, cfg.min_data_in_bin,
                           filter_cnt, cfg.feature_pre_filter, cfg.use_missing, cfg.zero_as_missing, is_cat);
      }
      row_off += ln;
    }
    inner_of.assign(F, -1);
    for (int f = 0; f < F; ++f) if (!mappers[f].is_trivial) { inner_of[f] = static_cast<int>(used.size()); used.push_back(f); }
    alloc_bins();
#pragma omp parallel for schedule(static)
    for (int u = 0; u < static_cast<int>(used.size()); ++u) {
      int f = used[u];
      if (wide) { uint16_t* col = &bins16[static_cast<size_t>(u) * n]; for (int i = 0; i < n; ++i) col[i] = static_cast<uint16_t>(mappers[f].ValueToBin(X[static_cast<size_t>(i) * F + f])); }
      else { uint8_t* col = &bins[static_cast<size_t>(u) * n]; for (int i = 0; i < n; ++i) col[i] = static_cast<uint8_t>(mappers[f].ValueToBin(X[static_cast<size_t>(i) * F + f])); }
    }
    feature_names.resize(F);
    for (int f = 0; f < F; ++f) feature_names[f] = "Column_" + std::to_string(f);
  }
};

// ------------------------------------------------------------------ objectives [UPSTREAM src/objective/*.hpp]
struct Objective {
  const Dataset* ds = nullptr;
  Config cfg;
  std::string name;
  int num_tree_per_iter = 1;
  bool need_train = true;
  virtual ~Objective() {}
  virtual void Init(const Dataset* d, const Config& c) { ds = d; cfg = c; }
  virtual void GetGradients(const double* score, float* g, float* h) const = 0;
  virtual double BoostFromScore(int class_id, int r0, int r1) const = 0;   // over rows [r0,r1) (one rank's shard)
  virtual bool IsConstantHessian() const { return false; }
  virtual bool ClassNeedTrain(int) const { return true; }
  virtual std::string ToString() const = 0;
  virtual bool GlobalInitScore() const { return false; }   // true: BoostFromScore already syncs sums across ranks
  // objectives whose leaf outputs are re-fitted after the tree is grown (L1 / quantile / MAPE)  [LightGBM IsRenewTreeOutput]
  virtual bool IsRenewTreeOutput() const { return false; }
  // rows = the leaf's (in-bag) rows of ONE rank, in partition order; residual(i) = label[i] - score[i]
  virtual double RenewTreeOutput(const std::vector<int>&, const std::function<double(int)>&) const { return 0.0; }
};

// [LightGBM src/objective/regression_objective.hpp PercentileFun / WeightedPercentileFun]
// percentile at `alpha` counted from the TOP of the descending order d[]: float position fp = (cnt-1)(1-alpha), linear interpolation
// between d[int(fp)] and d[int(fp)+1] (LightGBM >= 3.0: pos = int(fp) + 1, bias = fp - (pos - 1)); median of {1,2,3,4} = 2.5
template <typename T, typename Reader>
static T PercentileOf(Reader data_reader, int cnt, double alpha) {
  if (cnt <= 1) return data_reader(0);
  std::vector<T> ref(cnt);
  for (int i = 0; i < cnt; ++i) ref[i] = data_reader(i);
  const double float_pos = static_cast<double>(cnt - 1) * (1.0 - alpha);
  const int pos = static_cast<int>(float_pos) + 1;
  if (pos < 1) return *std::max_element(ref.begin(), ref.end());
  if (pos >= cnt) return *std::min_element(ref.begin(), ref.end());
  const double bias = float_pos - (pos - 1);
  std::sort(ref.begin(), ref.end(), std::greater<T>());
  const T v1 = ref[pos - 1], v2 = ref[pos];
  return static_cast<T>(v1 - (v1 - v2) * bias);
}
template <typename T, typename Reader, typename WReader>
static T WeightedPercentileOf(Reader data_reader, WReader weight_reader, int cnt, double alpha) {
  if (cnt <= 1) return data_reader(0);
  std::vector<int> sorted_idx(cnt);
  std::iota(sorted_idx.begin(), sorted_idx.end(), 0);
  std::stable_sort(sorted_idx.begin(), sorted_idx.end(), [&](int a, int b) { return data_reader(a) < data_reader(b); });
  std::vector<double> cdf(cnt);
  cdf[0] = weight_reader(sorted_idx[0]);
  for (int i = 1; i < cnt; ++i) cdf[i] = cdf[i - 1] + weight_reader(sorted_idx[i]);
  const double threshold = cdf[cnt - 1] * alpha;
  size_t pos = std::upper_bound(cdf.begin(), cdf.end(), threshold) - cdf.begin();
  pos = std::min(pos, static_cast<size_t>(cnt - 1));
  if (pos == 0 || pos == static_cast<size_t>(cnt - 1)) return data_reader(sorted_idx[pos]);
  const T v1 = data_reader(sorted_idx[pos - 1]), v2 = data_reader(sorted_idx[pos]);
  if (cdf[pos + 1] - cdf[pos] >= 1.0f) return static_cast<T>((threshold - cdf[pos]) / (cdf[pos + 1] - cdf[pos]) * (v2 - v1) + v1);
  return static_cast<T>(v2);
}

struct RegressionL2 : Objective {
  void GetGradients(const double* score, float* g, float* h) const override {
    const int n = ds->n;
    const float* y = ds->label.data();
    if (ds->weight.empty()) {
#pragma omp parallel for schedule(static)
      for (int i = 0; i < n; ++i) { g[i] = static_cast<float>(score[i] - y[i]); h[i] = 1.0f; }
    } else {
      const float* w = ds->weight.data();
#pragma omp parallel for schedule(static)
      for (int i = 0; i < n; ++i) { g[i] = static_cast<float>((score[i] - y[i]) * w[i]); h[i] = w[i]; }
    }
  }
  double BoostFromScore(int, int r0, int r1) const override {
    double suml = 0, sumw = 0;
    if (!ds->weight.empty()) { for (int i = r0; i < r1; ++i) { suml += static_cast<double>(ds->label[i]) * ds->weight[i]; sumw += ds->weight[i]; } }
    else { sumw = r1 - r0; for (int i = r0; i < r1; ++i) suml += ds->label[i]; }
    return suml / sumw;
  }
  bool IsConstantHessian() const override { return ds->weight.empty(); }
  std::string ToString() const override { return "regression"; }
};

// [UPSTREAM regression_objective.hpp] huber / fair / poisson / gamma / tweedie: elementwise variants of L2
struct RegressionVariant : RegressionL2 {
  int kind;   // 1 huber, 2 fair, 3 poisson, 4 gamma, 5 tweedie
  explicit RegressionVariant(int k) : kind(k) {}
  void GetGradients(const double* score, float* g, float* h) const override {
    const int n = ds->n;
    const float* y = ds->label.data();
    const float* w = ds->weight.empty() ? nullptr : ds->weight.data();
    const double alpha = cfg.alpha, c = cfg.fair_c, mds = cfg.poisson_max_delta_step, rho = cfg.tweedie_variance_power;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
      double gg, hh;
      const double s = score[i], lab = y[i];
      if (kind == 1) { const double diff = s - lab; gg = std::fabs(diff) <= alpha ? diff : ((diff > 0.0) - (diff < 0.0)) * alpha; hh = 1.0; }
      else if (kind == 2) { const double x = s - lab; gg = c * x / (std::fabs(x) + c); hh = c * c / ((std::fabs(x) + c) * (std::fabs(x) + c)); }
      else if (kind == 3) { gg = std::exp(s) - lab; hh = std::exp(s + mds); }
      else if (kind == 4) { gg = 1.0 - lab * std::exp(-s); hh = lab * std::exp(-s); }
      else { gg = -lab * std::exp((1 - rho) * s) + std::exp((2 - rho) * s); hh = -lab * (1 - rho) * std::exp((1 - rho) * s) + (2 - rho) * std::exp((2 - rho) * s); }
      if (w) { gg *= w[i]; hh *= w[i]; }
      g[i] = static_cast<float>(gg); h[i] = static_cast<float>(hh);
    }
  }
  double BoostFromScore(int k, int r0, int r1) const override {
    double m = RegressionL2::BoostFromScore(k, r0, r1);
    if (kind >= 3) return m > 0 ? std::log(m) : -std::numeric_limits<double>::infinity();
    return m;
  }
  bool IsConstantHessian() const override { return false; }
  std::string ToString() const override {
    static const char* names[] = {"", "huber", "fair", "poisson", "gamma", "tweedie"};
    return names[kind];
  }
};

// [LightGBM regression_objective.hpp RegressionL1loss / RegressionQuantileloss / RegressionMAPELOSS]
struct RegressionPercentile : RegressionL2 {
  int kind;                 // 0 l1, 1 quantile, 2 mape
  float alpha_f = 0.5f;     // quantile keeps alpha as score_t
  std::vector<float> label_weight;      // mape: 1 / max(1, |label|) (* weight)
  explicit RegressionPercentile(int k) : kind(k) {}
  void Init(const Dataset* d, const Config& c) override {
    Objective::Init(d, c);
    alpha_f = static_cast<float>(c.alpha);
    if (kind == 2) {
      label_weight.resize(d->n);
      for (int i = 0; i < d->n; ++i) {
        label_weight[i] = 1.0f / std::max(1.0f, std::fabs(d->label[i]));
        if (!d->weight.empty()) label_weight[i] *= d->weight[i];
      }
    }
  }
  double Alpha() const { return kind == 1 ? static_cast<double>(alpha_f) : 0.5; }
  void GetGradients(const double* score, float* g, float* h) const override {
    const int n = ds->n;
    const float* y = ds->label.data();
    const float* w = ds->weight.empty() ? nullptr : ds->weight.data();
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
      if (kind == 1) {
        const float delta = static_cast<float>(score[i] - y[i]);
        const float gg = delta >= 0 ? (1.0f - alpha_f) : -alpha_f;
        g[i] = w ? static_cast<float>(gg * w[i]) : gg;
        h[i] = w ? w[i] : 1.0f;
      } else {
        const double diff = score[i] - y[i];
        const int sgn = (diff > 0.0) - (diff < 0.0);
        if (kind == 0) { g[i] = w ? static_cast<float>(sgn * w[i]) : static_cast<float>(sgn); h[i] = w ? w[i] : 1.0f; }
        else { g[i] = static_cast<float>(sgn * label_weight[i]); h[i] = w ? w[i] : 1.0f; }
      }
    }
  }
  double BoostFromScore(int, int r0, int r1) const override {
    const float* y = ds->label.data();
    const int cnt = r1 - r0;
    if (kind == 2) return WeightedPercentileOf<float>([&](int i) { return y[r0 + i]; }, [&](int i) { return label_weight[r0 + i]; }, cnt, 0.5);
    if (ds->weight.empty()) return PercentileOf<float>([&](int i) { return y[r0 + i]; }, cnt, Alpha());
    return WeightedPercentileOf<float>([&](int i) { return y[r0 + i]; }, [&](int i) { return ds->weight[r0 + i]; }, cnt, Alpha());
  }
  bool IsRenewTreeOutput() const override { return true; }
  double RenewTreeOutput(const std::vector<int>& rows, const std::function<double(int)>& residual) const override {
    const int cnt = static_cast<int>(rows.size());
    auto dr = [&](int i) { return residual(rows[i]); };
    if (kind == 2) return WeightedPercentileOf<double>(dr, [&](int i) { return label_weight[rows[i]]; }, cnt, 0.5);
    if (ds->weight.empty()) return PercentileOf<double>(dr, cnt, Alpha());
    return WeightedPercentileOf<double>(dr, [&](int i) { return ds->weight[rows[i]]; }, cnt, Alpha());
  }
  bool IsConstantHessian() const override { return ds->weight.empty(); }
  std::string ToString() const override { return kind == 0 ? "regression_l1" : kind == 1 ? "quantile" : "mape"; }
};

struct BinaryLogloss : Objective {
  double label_weights[2] = {1.0, 1.0};
  void Init(const Dataset* d, const Config& c) override {
    Objective::Init(d, c);
    long cnt_pos = 0, cnt_neg = 0;
    for (int i = 0; i < d->n; ++i) { if (d->label[i] > 0) ++cnt_pos; else ++cnt_neg; }
    need_train = !(cnt_neg == 0 || cnt_pos == 0);     // counts are global (summed over ranks) [UPSTREAM]
    if (c.is_unbalance && cnt_pos > 0 && cnt_neg > 0) {
      if (cnt_pos > cnt_neg) { label_weights[1] = 1.0; label_weights[0] = static_cast<double>(cnt_pos) / cnt_neg; }
      else { label_weights[1] = static_cast<double>(cnt_neg) / cnt_pos; label_weights[0] = 1.0; }
    }
    label_weights[1] *= c.scale_pos_weight;
  }
  void GetGradients(const double* score, float* g, float* h) const override {
    if (!need_train) return;
    const int n = ds->n;
    const double sig = cfg.sigmoid;
    const float* y = ds->label.data();
    const float* w = ds->weight.empty() ? nullptr : ds->weight.data();
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
      const int is_pos = y[i] > 0;
      const int label = is_pos ? 1 : -1;
      const double lw = label_weights[is_pos];
      const double response = -label * sig / (1.0 + std::exp(label * sig * score[i]));
      const double abs_response = std::fabs(response);
      if (!w) { g[i] = static_cast<float>(response * lw); h[i] = static_cast<float>(abs_response * (sig - abs_response) * lw); }
      else { g[i] = static_cast<float>(response * lw * w[i]); h[i] = static_cast<float>(abs_response * (sig - abs_response) * lw * w[i]); }
    }
  }
  double BoostFromScore(int, int, int) const override {   // sums synced over ranks => global
    double suml = 0, sumw = 0;
    const int n = ds->n;
    if (!ds->weight.empty()) { for (int i = 0; i < n; ++i) { suml += (ds->label[i] > 0) * static_cast<double>(ds->weight[i]); sumw += ds->weight[i]; } }
    else { sumw = n; for (int i = 0; i < n; ++i) suml += (ds->label[i] > 0); }
    double pavg = suml / sumw;
    pavg = std::min(pavg, 1.0 - kEpsilon);
    pavg = std::max(pavg, kEpsilon);
    return std::log(pavg / (1.0 - pavg)) / cfg.sigmoid;
  }
  bool GlobalInitScore() const override { return true; }
  bool ClassNeedTrain(int) const override { return need_train; }
  std::string ToString() const override {
    std::ostringstream s; s << "binary sigmoid:" << cfg.sigmoid; return s.str();
  }
};

struct MulticlassSoftmax : Objective {
  int K = 1;
  double factor = 1.0;
  std::vector<int> label_int;
  std::vector<double> class_init_probs;
  void Init(const Dataset* d, const Config& c) override {
    Objective::Init(d, c);
    K = c.num_class; num_tree_per_iter = K;
    factor = static_cast<double>(K) / (K - 1.0);
    label_int.resize(d->n);
    class_init_probs.assign(K, 0.0);
    double sum_weight = 0;
    for (int i = 0; i < d->n; ++i) {
      label_int[i] = static_cast<int>(d->label[i]);
      double w = d->weight.empty() ? 1.0 : d->weight[i];
      class_init_probs[label_int[i]] += w; sum_weight += w;
    }
    for (int k = 0; k < K; ++k) class_init_probs[k] /= sum_weight;
  }
  void GetGradients(const double* score, float* g, float* h) const override {
    const int n = ds->n;
    const float* w = ds->weight.empty() ? nullptr : ds->weight.data();
#pragma omp parallel
    {
      std::vector<double> rec(K);
#pragma omp for schedule(static)
      for (int i = 0; i < n; ++i) {
        for (int k = 0; k < K; ++k) rec[k] = score[static_cast<size_t>(n) * k + i];
        double wmax = rec[0];
        for (int k = 1; k < K; ++k) wmax = std::max(rec[k], wmax);
        double wsum = 0;
        for (int k = 0; k < K; ++k) { rec[k] = std::exp(rec[k] - wmax); wsum += rec[k]; }
        for (int k = 0; k < K; ++k) rec[k] /= wsum;
        for (int k = 0; k < K; ++k) {
          double p = rec[k];
          size_t idx = static_cast<size_t>(n) * k + i;
          double gg = (label_int[i] == k) ? p - 1.0 : p;
          double hh = factor * p * (1.0 - p);
          if (w) { gg *= w[i]; hh *= w[i]; }
          g[idx] = static_cast<float>(gg); h[idx] = static_cast<float>(hh);
        }
      }
    }
  }
  double BoostFromScore(int k, int, int) const override { return std::log(std::max(kEpsilon, class_init_probs[k])); }
  bool GlobalInitScore() const override { return true; }
  bool ClassNeedTrain(int k) const override {
    return !(std::fabs(class_init_probs[k]) <= kEpsilon || std::fabs(class_init_probs[k]) >= 1.0 - kEpsilon);
  }
  std::string ToString() const override { return "multiclass num_class:" + std::to_string(K); }
};

// [UPSTREAM multiclass_objective.hpp MulticlassOVA]: num_class independent BinaryLogloss objectives, class k's labels = (label == k)
struct MulticlassOVA : Objective {
  int K = 1;
  std::vector<double> w_neg, w_pos;       // BinaryLogloss::label_weights_ per class
  std::vector<char> class_need_train;
  void Init(const Dataset* d, const Config& c) override {
    Objective::Init(d, c);
    K = c.num_class; num_tree_per_iter = K;
    w_neg.assign(K, 1.0); w_pos.assign(K, 1.0); class_need_train.assign(K, 1);
    for (int k = 0; k < K; ++k) {
      long cnt_pos = 0, cnt_neg = 0;
      for (int i = 0; i < d->n; ++i) { if (static_cast<int>(d->label[i]) == k) ++cnt_pos; else ++cnt_neg; }
      class_need_train[k] = !(cnt_neg == 0 || cnt_pos == 0);
      if (c.is_unbalance && cnt_pos > 0 && cnt_neg > 0) {
        if (cnt_pos > cnt_neg) { w_pos[k] = 1.0; w_neg[k] = static_cast<double>(cnt_pos) / cnt_neg; }
        else { w_pos[k] = static_cast<double>(cnt_neg) / cnt_pos; w_neg[k] = 1.0; }
      }
      w_pos[k] *= c.scale_pos_weight;
    }
  }
  void GetGradients(const double* score, float* g, float* h) const override {
    const int n = ds->n;
    const double sig = cfg.sigmoid;
    const float* y = ds->label.data();
    const float* w = ds->weight.empty() ? nullptr : ds->weight.data();
    for (int k = 0; k < K; ++k) {
      if (!class_need_train[k]) continue;
      const size_t off = static_cast<size_t>(n) * k;
#pragma omp parallel for schedule(static)
      for (int i = 0; i < n; ++i) {
        const int is_pos = static_cast<int>(y[i]) == k;
        const int label = is_pos ? 1 : -1;
        const double lw = is_pos ? w_pos[k] : w_neg[k];
        const double response = -label * sig / (1.0 + std::exp(label * sig * score[off + i]));
        const double abs_response = std::fabs(response);
        if (!w) { g[off + i] = static_cast<float>(response * lw); h[off + i] = static_cast<float>(abs_response * (sig - abs_response) * lw); }
        else { g[off + i] = static_cast<float>(response * lw * w[i]); h[off + i] = static_cast<float>(abs_response * (sig - abs_response) * lw * w[i]); }
      }
    }
  }
  double BoostFromScore(int k, int, int) const override {
    double suml = 0, sumw = 0;
    const int n = ds->n;
    if (!ds->weight.empty()) { for (int i = 0; i < n; ++i) { suml += (static_cast<int>(ds->label[i]) == k) * static_cast<double>(ds->weight[i]); sumw += ds->weight[i]; } }
    else { sumw = n; for (int i = 0; i < n; ++i) suml += (static_cast<int>(ds->label[i]) == k); }
    double pavg = suml / sumw;
    pavg = std::min(pavg, 1.0 - kEpsilon);
    pavg = std::max(pavg, kEpsilon);
    return std::log(pavg / (1.0 - pavg)) / cfg.sigmoid;
  }
  bool GlobalInitScore() const override { return true; }
  bool ClassNeedTrain(int k) const override { return class_need_train[k] != 0; }
  std::string ToString() const override {
    std::ostringstream s; s << "multiclassova num_class:" << K << " sigmoid:" << cfg.sigmoid; return s.str();
  }
};

// [UPSTREAM xentropy_objective.hpp CrossEntropy]: labels are probabilities in [0, 1]
struct CrossEntropy : Objective {
  void GetGradients(const double* score, float* g, float* h) const override {
    const int n = ds->n;
    const float* y = ds->label.data();
    const float* w = ds->weight.empty() ? nullptr : ds->weight.data();
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
      const double z = 1.0 / (1.0 + std::exp(-score[i]));
      if (!w) { g[i] = static_cast<float>(z - y[i]); h[i] = static_cast<float>(z * (1.0 - z)); }
      else { g[i] = static_cast<float>((z - y[i]) * w[i]); h[i] = static_cast<float>(z * (1.0 - z) * w[i]); }
    }
  }
  double BoostFromScore(int, int, int) const override {
    double suml = 0, sumw = 0;
    const int n = ds->n;
    if (!ds->weight.empty()) { for (int i = 0; i < n; ++i) { suml += static_cast<double>(ds->label[i]) * ds->weight[i]; sumw += ds->weight[i]; } }
    else { sumw = n; for (int i = 0; i < n; ++i) suml += ds->label[i]; }
    double pavg = suml / sumw;
    pavg = std::min(pavg, 1.0 - kEpsilon);
    pavg = std::max(pavg, kEpsilon);
    return std::log(pavg / (1.0 - pavg));
  }
  bool GlobalInitScore() const override { return true; }
  std::string ToString() const override { return "cross_entropy"; }
};

struct LambdarankNDCG : Objective {
  std::vector<double> label_gain, inverse_max_dcg, discount;
  std::vector<float> sigmoid_table;
  int truncation = 30;
  bool norm = true;
  double sig = 1.0, min_in = -50, max_in = 50, idx_factor = 0;
  static constexpr size_t kSigBins = 1024 * 1024;
  void Init(const Dataset* d, const Config& c) override {
    Objective::Init(d, c);
    sig = c.sigmoid; truncation = c.lambdarank_truncation_level; norm = c.lambdarank_norm;
    label_gain = c.label_gain;
    if (label_gain.empty()) { label_gain.push_back(0.0); for (int i = 1; i < 31; ++i) label_gain.push_back(static_cast<double>((1 << i) - 1)); }
    int maxq = 0;
    int nq = static_cast<int>(d->query_boundaries.size()) - 1;
    for (int q = 0; q < nq; ++q) maxq = std::max(maxq, d->query_boundaries[q + 1] - d->query_boundaries[q]);
    discount.resize(std::max(maxq, 10000) + 1);
    for (size_t i = 0; i < discount.size(); ++i) discount[i] = 1.0 / std::log2(2.0 + i);
    inverse_max_dcg.resize(nq);
    for (int q = 0; q < nq; ++q) {
      int s = d->query_boundaries[q], cnt = d->query_boundaries[q + 1] - s;
      double m = MaxDCGAtK(truncation, d->label.data() + s, cnt);
      inverse_max_dcg[q] = m > 0.0 ? 1.0 / m : m;
    }
    min_in = min_in / sig / 2; max_in = max_in / sig / 2;
    sigmoid_table.resize(kSigBins);
    idx_factor = kSigBins / (max_in - min_in);
    for (size_t i = 0; i < kSigBins; ++i) {
      double score = i / idx_factor + min_in;
      sigmoid_table[i] = static_cast<float>(1.0 / (1.0 + std::exp(score * sig)));
    }
  }
  double MaxDCGAtK(int k, const float* label, int num) const {
    std::vector<int> label_cnt(label_gain.size(), 0);
    for (int i = 0; i < num; ++i) ++label_cnt[static_cast<int>(label[i])];
    int top = static_cast<int>(label_gain.size()) - 1;
    if (k > num) k = num;
    double ret = 0;
    for (int j = 0; j < k; ++j) {
      while (top > 0 && label_cnt[top] <= 0) --top;
      if (top < 0) break;
      ret += discount[j] * label_gain[top];
      --label_cnt[top];
    }
    return ret;
  }
  double GetSigmoid(double s) const {
    if (s <= min_in) return sigmoid_table[0];
    if (s >= max_in) return sigmoid_table[kSigBins - 1];
    return sigmoid_table[static_cast<size_t>((s - min_in) * idx_factor)];
  }
  void OneQuery(int q, int cnt, const float* label, const double* score, float* lambdas, float* hessians) const {
    const double imd = inverse_max_dcg[q];
    for (int i = 0; i < cnt; ++i) { lambdas[i] = 0.0f; hessians[i] = 0.0f; }
    std::vector<int> sorted(cnt);
    std::iota(sorted.begin(), sorted.end(), 0);
    std::stable_sort(sorted.begin(), sorted.end(), [score](int a, int b) { return score[a] > score[b]; });
    const double best_score = score[sorted[0]];
    int worst_idx = cnt - 1;
    if (worst_idx > 0 && score[sorted[worst_idx]] == kMinScore) worst_idx -= 1;
    const double worst_score = score[sorted[worst_idx]];
    double sum_lambdas = 0.0;
    for (int i = 0; i < cnt - 1 && i < truncation; ++i) {
      if (score[sorted[i]] == kMinScore) continue;
      for (int j = i + 1; j < cnt; ++j) {
        if (score[sorted[j]] == kMinScore) continue;
        if (label[sorted[i]] == label[sorted[j]]) continue;
        int high_rank, low_rank;
        if (label[sorted[i]] > label[sorted[j]]) { high_rank = i; low_rank = j; } else { high_rank = j; low_rank = i; }
        const int high = sorted[high_rank], low = sorted[low_rank];
        const double delta_score = score[high] - score[low];
        const double dcg_gap = label_gain[static_cast<int>(label[high])] - label_gain[static_cast<int>(label[low])];
        const double paired_discount = std::fabs(discount[high_rank] - discount[low_rank]);
        double delta_pair_NDCG = dcg_gap * paired_discount * imd;
        if (norm && best_score != worst_score) delta_pair_NDCG /= (0.01f + std::fabs(delta_score));
        double p_lambda = GetSigmoid(delta_score);
        double p_hessian = p_lambda * (1.0f - p_lambda);
        p_lambda *= -sig * delta_pair_NDCG;
        p_hessian *= sig * sig * delta_pair_NDCG;
        lambdas[low] -= static_cast<float>(p_lambda);
        hessians[low] += static_cast<float>(p_hessian);
        lambdas[high] += static_cast<float>(p_lambda);
        hessians[high] += static_cast<float>(p_hessian);
        sum_lambdas -= 2 * p_lambda;
      }
    }
    if (norm && sum_lambdas > 0) {
      double nf = std::log2(1 + sum_lambdas) / sum_lambdas;
      for (int i = 0; i < cnt; ++i) { lambdas[i] = static_cast<float>(lambdas[i] * nf); hessians[i] = static_cast<float>(hessians[i] * nf); }
    }
  }
  void GetGradients(const double* score, float* g, float* h) const override {
    int nq = static_cast<int>(ds->query_boundaries.size()) - 1;
#pragma omp parallel for schedule(guided)
    for (int q = 0; q < nq; ++q) {
      int s = ds->query_boundaries[q], cnt = ds->query_boundaries[q + 1] - s;
      OneQuery(q, cnt, ds->label.data() + s, score + s, g + s, h + s);
      if (!ds->weight.empty())
        for (int j = 0; j < cnt; ++j) { g[s + j] = static_cast<float>(g[s + j] * ds->weight[s + j]); h[s + j] = static_cast<float>(h[s + j] * ds->weight[s + j]); }
    }
  }
  double BoostFromScore(int, int, int) const override { return 0.0; }
  std::string ToString() const override { return "lambdarank"; }
};

static Objective* CreateObjective(const Config& c) {
  if (c.objective == "regression") return new RegressionL2();
  if (c.objective == "huber") return new RegressionVariant(1);
  if (c.objective == "fair") return new RegressionVariant(2);
  if (c.objective == "poisson") return new RegressionVariant(3);
  if (c.objective == "gamma") return new RegressionVariant(4);
  if (c.objective == "tweedie") return new RegressionVariant(5);
  if (c.objective == "regression_l1") return new RegressionPercentile(0);
  if (c.objective == "quantile") return new RegressionPercentile(1);
  if (c.objective == "mape") return new RegressionPercentile(2);
  if (c.objective == "binary") return new BinaryLogloss();
  if (c.objective == "multiclass") return new MulticlassSoftmax();
  if (c.objective == "multiclassova") return new MulticlassOVA();
  if (c.objective == "cross_entropy") return new CrossEntropy();
  if (c.objective == "lambdarank") return new LambdarankNDCG();
  return nullptr;
}

// ------------------------------------------------------------------ split finding [UPSTREAM treelearner/feature_histogram.hpp]
struct SplitInfo {
  int feature = -1;            // real feature index
  uint32_t threshold = 0;
  int left_count = 0, right_count = 0;
  double left_output = 0, right_output = 0;
  double gain = kMinScore;
  double left_sum_gradient = 0, left_sum_hessian = 0, right_sum_gradient = 0, right_sum_hessian = 0;
  bool default_left = true;
  std::vector<uint32_t> cat_threshold;   // categorical split: bins that go LEFT
  bool better_than(const SplitInfo& o) const {     // operator>
    double lg = gain, og = o.gain;
    if (std::isnan(lg)) lg = kMinScore;
    if (std::isnan(og)) og = kMinScore;
    int lf = feature == -1 ? INT32_MAX : feature, of = o.feature == -1 ? INT32_MAX : o.feature;
    if (lg != og) return lg > og;
    return lf < of;
  }
};

inline double Sign(double x) { return (x > 0.0) - (x < 0.0); }
inline double ThresholdL1(double s, double l1) { double r = std::max(0.0, std::fabs(s) - l1); return Sign(s) * r; }
inline int RoundInt(double x) { return static_cast<int>(x + 0.5); }

struct SplitCfg { double l1, l2, max_delta_step, min_gain_to_split, min_sum_hessian; int min_data_in_leaf;
                  int max_cat_threshold = 32, max_cat_to_onehot = 4, min_data_per_group = 100; double cat_l2 = 10.0, cat_smooth = 10.0; };

inline double CalcOutput(double g, double h, const SplitCfg& c) {
  double ret = (c.l1 > 0) ? -ThresholdL1(g, c.l1) / (h + c.l2) : -g / (h + c.l2);
  if (c.max_delta_step > 0 && std::fabs(ret) > c.max_delta_step) ret = Sign(ret) * c.max_delta_step;
  return ret;
}
inline double LeafGainGivenOutput(double g, double h, const SplitCfg& c, double out) {
  double sg = (c.l1 > 0) ? ThresholdL1(g, c.l1) : g;
  return -(2.0 * sg * out + (h + c.l2) * out * out);
}
inline double LeafGain(double g, double h, const SplitCfg& c) {
  if (!(c.max_delta_step > 0)) {
    if (c.l1 > 0) { double sg = ThresholdL1(g, c.l1); return (sg * sg) / (h + c.l2); }
    return (g * g) / (h + c.l2);
  }
  return LeafGainGivenOutput(g, h, c, CalcOutput(g, h, c));
}

// hist: direct accumulation, entry b = feature bin b, interleaved (g,h).  `offset` = (most_freq_bin==0)
// reproduces the upstream storage convention data_[t] == bin t+offset.
struct ScanMeta { int num_bin; int missing_type; int default_bin; int offset; };

template <bool REVERSE, bool SKIP_DEFAULT_BIN, bool NA_AS_MISSING>
static void ScanSequential(const double* hist, const ScanMeta& m, const SplitCfg& c, double sum_gradient, double sum_hessian,
                           int num_data, double min_gain_shift, SplitInfo* output, bool* is_splittable) {
  const int offset = m.offset;
  auto GRAD = [&](int t) { return hist[(t + offset) * 2]; };
  auto HESS = [&](int t) { return hist[(t + offset) * 2 + 1]; };
  double best_sum_left_gradient = NAN, best_sum_left_hessian = NAN, best_gain = kMinScore;
  int best_left_count = 0;
  uint32_t best_threshold = static_cast<uint32_t>(m.num_bin);
  const double cnt_factor = num_data / sum_hessian;
  if (REVERSE) {
    double sum_right_gradient = 0.0, sum_right_hessian = kEpsilon;
    int right_count = 0;
    int t = m.num_bin - 1 - offset - NA_AS_MISSING;
    const int t_end = 1 - offset;
    for (; t >= t_end; --t) {
      if (SKIP_DEFAULT_BIN && (t + offset) == m.default_bin) continue;
      const double grad = GRAD(t), hess = HESS(t);
      int cnt = RoundInt(hess * cnt_factor);
      sum_right_gradient += grad; sum_right_hessian += hess; right_count += cnt;
      if (right_count < c.min_data_in_leaf || sum_right_hessian < c.min_sum_hessian) continue;
      int left_count = num_data - right_count;
      if (left_count < c.min_data_in_leaf) break;
      double sum_left_hessian = sum_hessian - sum_right_hessian;
      if (sum_left_hessian < c.min_sum_hessian) break;
      double sum_left_gradient = sum_gradient - sum_right_gradient;
      double current_gain = LeafGain(sum_left_gradient, sum_left_hessian, c) + LeafGain(sum_right_gradient, sum_right_hessian, c);
      if (current_gain <= min_gain_shift) continue;
      *is_splittable = true;
      if (current_gain > best_gain) {
        best_left_count = left_count; best_sum_left_gradient = sum_left_gradient; best_sum_left_hessian = sum_left_hessian;
        best_threshold = static_cast<uint32_t>(t - 1 + offset); best_gain = current_gain;
      }
    }
  } else {
    double sum_left_gradient = 0.0, sum_left_hessian = kEpsilon;
    int left_count = 0;
    int t = 0;
    const int t_end = m.num_bin - 2 - offset;
    if (NA_AS_MISSING && offset == 1) {
      sum_left_gradient = sum_gradient; sum_left_hessian = sum_hessian - kEpsilon; left_count = num_data;
      for (int i = 0; i < m.num_bin - offset; ++i) {
        const double grad = GRAD(i), hess = HESS(i);
        int cnt = RoundInt(hess * cnt_factor);
        sum_left_gradient -= grad; sum_left_hessian -= hess; left_count -= cnt;
      }
      t = -1;
    }
    for (; t <= t_end; ++t) {
      if (SKIP_DEFAULT_BIN && (t + offset) == m.default_bin) continue;
      if (t >= 0) {
        sum_left_gradient += GRAD(t); sum_left_hessian += HESS(t);
        left_count += RoundInt(HESS(t) * cnt_factor);
      }
      if (left_count < c.min_data_in_leaf || sum_left_hessian < c.min_sum_hessian) continue;
      int right_count = num_data - left_count;
      if (right_count < c.min_data_in_leaf) break;
      double sum_right_hessian = sum_hessian - sum_left_hessian;
      if (sum_right_hessian < c.min_sum_hessian) break;
      double sum_right_gradient = sum_gradient - sum_left_gradient;
      double current_gain = LeafGain(sum_left_gradient, sum_left_hessian, c) + LeafGain(sum_right_gradient, sum_right_hessian, c);
      if (current_gain <= min_gain_shift) continue;
      *is_splittable = true;
      if (current_gain > best_gain) {
        best_left_count = left_count; best_sum_left_gradient = sum_left_gradient; best_sum_left_hessian = sum_left_hessian;
        best_threshold = static_cast<uint32_t>(t + offset); best_gain = current_gain;
      }
    }
  }
  if (*is_splittable && best_gain > output->gain + min_gain_shift) {
    output->threshold = best_threshold;
    output->left_output = CalcOutput(best_sum_left_gradient, best_sum_left_hessian, c);
    output->left_count = best_left_count;
    output->left_sum_gradient = best_sum_left_gradient;
    output->left_sum_hessian = best_sum_left_hessian - kEpsilon;
    output->right_output = CalcOutput(sum_gradient - best_sum_left_gradient, sum_hessian - best_sum_left_hessian, c);
    output->right_count = num_data - best_left_count;
    output->right_sum_gradient = sum_gradient - best_sum_left_gradient;
    output->right_sum_hessian = sum_hessian - best_sum_left_hessian - kEpsilon;
    output->gain = best_gain - min_gain_shift;
    output->default_left = REVERSE;
  }
}

// FeatureHistogram::FindBestThreshold (numerical)
static void FindBestThresholdNumerical(const double* hist, const ScanMeta& m, const SplitCfg& c, double sum_gradient,
                                       double sum_hessian_in, int num_data, SplitInfo* out, bool* is_splittable) {
  out->default_left = true;
  out->gain = kMinScore;
  double sum_hessian = sum_hessian_in + 2 * kEpsilon;
  *is_splittable = false;
  double min_gain_shift = LeafGain(sum_gradient, sum_hessian, c) + c.min_gain_to_split;
  if (m.num_bin > 2 && m.missing_type != kMissNone) {
    if (m.missing_type == kMissZero) {
      ScanSequential<true, true, false>(hist, m, c, sum_gradient, sum_hessian, num_data, min_gain_shift, out, is_splittable);
      ScanSequential<false, true, false>(hist, m, c, sum_gradient, sum_hessian, num_data, min_gain_shift, out, is_splittable);
    } else {
      ScanSequential<true, false, true>(hist, m, c, sum_gradient, sum_hessian, num_data, min_gain_shift, out, is_splittable);
      ScanSequential<false, false, true>(hist, m, c, sum_gradient, sum_hessian, num_data, min_gain_shift, out, is_splittable);
    }
  } else {
    ScanSequential<true, false, false>(hist, m, c, sum_gradient, sum_hessian, num_data, min_gain_shift, out, is_splittable);
    if (m.missing_type == kMissNaN) out->default_left = false;
  }
}

// FeatureHistogram::FindBestThresholdCategoricalInner [UPSTREAM]: one-hot for <= max_cat_to_onehot bins, otherwise bins with
// enough data sorted by g/(h+cat_smooth) and scanned from both ends (many-vs-many), lambda_l2 += cat_l2.
static void FindBestThresholdCategorical(const double* hist, const ScanMeta& m, const SplitCfg& c0, double sum_gradient, double sum_hessian_in,
                                         int num_data, SplitInfo* output, bool* is_splittable) {
  output->default_left = false;
  output->gain = kMinScore;
  const double sum_hessian = sum_hessian_in + 2 * kEpsilon;
  *is_splittable = false;
  double best_gain = kMinScore, best_sum_left_gradient = 0, best_sum_left_hessian = 0;
  int best_left_count = 0;
  SplitCfg c = c0;
  SplitCfg cshift = c0; cshift.max_delta_step = 0;
  double gain_shift = (c0.max_delta_step > 0) ? LeafGainGivenOutput(sum_gradient, sum_hessian, c0, 0.0 /* parent_output unused w/o smoothing */)
                                              : LeafGain(sum_gradient, sum_hessian, cshift);
  if (c0.max_delta_step > 0) gain_shift = LeafGain(sum_gradient, sum_hessian, c0);
  const double min_gain_shift = gain_shift + c0.min_gain_to_split;
  auto GRAD = [&](int b) { return hist[b * 2]; };
  auto HESS = [&](int b) { return hist[b * 2 + 1]; };
  const bool use_onehot = m.num_bin <= c0.max_cat_to_onehot;
  int best_threshold = -1, best_dir = 1;
  const double cnt_factor = num_data / sum_hessian;
  std::vector<int> sorted_idx;
  int used_bin = -1;
  if (use_onehot) {
    for (int t = 1; t < m.num_bin; ++t) {
      const double grad = GRAD(t), hess = HESS(t);
      int cnt = RoundInt(hess * cnt_factor);
      if (cnt < c.min_data_in_leaf || hess < c.min_sum_hessian) continue;
      int other_count = num_data - cnt;
      if (other_count < c.min_data_in_leaf) continue;
      double sum_other_hessian = sum_hessian - hess - kEpsilon;
      if (sum_other_hessian < c.min_sum_hessian) continue;
      double sum_other_gradient = sum_gradient - grad;
      double current_gain = LeafGain(sum_other_gradient, sum_other_hessian, c) + LeafGain(grad, hess + kEpsilon, c);
      if (current_gain <= min_gain_shift) continue;
      *is_splittable = true;
      if (current_gain > best_gain) {
        best_threshold = t; best_sum_left_gradient = grad; best_sum_left_hessian = hess + kEpsilon; best_left_count = cnt; best_gain = current_gain;
      }
    }
  } else {
    for (int i = 1; i < m.num_bin; ++i) if (RoundInt(HESS(i) * cnt_factor) >= c.cat_smooth) sorted_idx.push_back(i);
    used_bin = static_cast<int>(sorted_idx.size());
    c.l2 += c.cat_l2;
    auto ctr = [&](int i) { return GRAD(i) / (HESS(i) + c.cat_smooth); };
    std::stable_sort(sorted_idx.begin(), sorted_idx.end(), [&](int i, int j) { return ctr(i) < ctr(j); });
    const int max_num_cat = std::min(c.max_cat_threshold, (used_bin + 1) / 2);
    const int dirs[2] = {1, -1};
    const int starts[2] = {0, used_bin - 1};
    for (int out_i = 0; out_i < 2; ++out_i) {
      int dir = dirs[out_i], start_pos = starts[out_i];
      int cnt_cur_group = 0, left_count = 0;
      double sum_left_gradient = 0.0, sum_left_hessian = kEpsilon;
      for (int i = 0; i < used_bin && i < max_num_cat; ++i) {
        int t = sorted_idx[start_pos];
        start_pos += dir;
        const double grad = GRAD(t), hess = HESS(t);
        int cnt = RoundInt(hess * cnt_factor);
        sum_left_gradient += grad; sum_left_hessian += hess; left_count += cnt; cnt_cur_group += cnt;
        if (left_count < c.min_data_in_leaf || sum_left_hessian < c.min_sum_hessian) continue;
        int right_count = num_data - left_count;
        if (right_count < c.min_data_in_leaf || right_count < c.min_data_per_group) break;
        double sum_right_hessian = sum_hessian - sum_left_hessian;
        if (sum_right_hessian < c.min_sum_hessian) break;
        if (cnt_cur_group < c.min_data_per_group) continue;
        cnt_cur_group = 0;
        double sum_right_gradient = sum_gradient - sum_left_gradient;
        double current_gain = LeafGain(sum_left_gradient, sum_left_hessian, c) + LeafGain(sum_right_gradient, sum_right_hessian, c);
        if (current_gain <= min_gain_shift) continue;
        *is_splittable = true;
        if (current_gain > best_gain) {
          best_left_count = left_count; best_sum_left_gradient = sum_left_gradient; best_sum_left_hessian = sum_left_hessian;
          best_threshold = i; best_gain = current_gain; best_dir = dir;
        }
      }
    }
  }
  if (*is_splittable) {
    output->left_output = CalcOutput(best_sum_left_gradient, best_sum_left_hessian, c);
    output->left_count = best_left_count;
    output->left_sum_gradient = best_sum_left_gradient;
    output->left_sum_hessian = best_sum_left_hessian - kEpsilon;
    output->right_output = CalcOutput(sum_gradient - best_sum_left_gradient, sum_hessian - best_sum_left_hessian, c);
    output->right_count = num_data - best_left_count;
    output->right_sum_gradient = sum_gradient - best_sum_left_gradient;
    output->right_sum_hessian = sum_hessian - best_sum_left_hessian - kEpsilon;
    output->gain = best_gain - min_gain_shift;
    output->cat_threshold.clear();
    if (use_onehot) output->cat_threshold.push_back(static_cast<uint32_t>(best_threshold));
    else {
      for (int i = 0; i <= best_threshold; ++i)
        output->cat_threshold.push_back(static_cast<uint32_t>(best_dir == 1 ? sorted_idx[i] : sorted_idx[used_bin - 1 - i]));
    }
    output->threshold = 0;
  }
}

inline std::vector<uint32_t> ConstructBitset(const std::vector<int>& vals) {
  std::vector<uint32_t> ret;
  for (int v : vals) {
    size_t i1 = static_cast<size_t>(v) / 32, i2 = static_cast<size_t>(v) % 32;
    if (ret.size() < i1 + 1) ret.resize(i1 + 1, 0);
    ret[i1] |= (1u << i2);
  }
  return ret;
}
inline bool FindInBitset(const uint32_t* bits, int n, int pos) {
  int i1 = pos / 32;
  if (pos < 0 || i1 >= n) return false;
  return (bits[i1] >> (pos % 32)) & 1;
}

// ------------------------------------------------------------------ tree [UPSTREAM io/tree.cpp]
inline double MaybeRoundToZero(double x) { return std::fabs(x) > kZeroThreshold ? x : 0.0; }
inline double AvoidInf(double x) {
  if (std::isnan(x)) return 0.0;
  if (x >= 1e300) return 1e300;
  if (x <= -1e300) return -1e300;
  return x;
}
struct Tree {
  int num_leaves = 1;
  int num_cat = 0;
  std::vector<int> cat_boundaries{0}, cat_boundaries_inner{0};
  std::vector<uint32_t> cat_threshold, cat_threshold_inner;
  double shrinkage = 1.0;
  std::vector<int> left_child, right_child, split_feature_inner, split_feature, leaf_parent, leaf_count, internal_count, leaf_depth;
  std::vector<uint32_t> threshold_in_bin;
  std::vector<double> threshold, leaf_value, leaf_weight, internal_value, internal_weight;
  std::vector<float> split_gain;
  std::vector<int8_t> decision_type;
  explicit Tree(int max_leaves) {
    int m = std::max(max_leaves, 2);
    left_child.assign(m - 1, 0); right_child.assign(m - 1, 0); split_feature_inner.assign(m - 1, 0);
    split_feature.assign(m - 1, 0); threshold_in_bin.assign(m - 1, 0); threshold.assign(m - 1, 0);
    decision_type.assign(m - 1, 0); split_gain.assign(m - 1, 0); leaf_parent.assign(m, -1);
    leaf_value.assign(m, 0); leaf_weight.assign(m, 0); leaf_count.assign(m, 0); internal_value.assign(m - 1, 0);
    internal_weight.assign(m - 1, 0); internal_count.assign(m - 1, 0); leaf_depth.assign(m, 0);
    leaf_depth[0] = 0; leaf_parent[0] = -1;
  }
  int Split(int leaf, int feature, int real_feature, uint32_t thr_bin, double thr_double, double left_value, double right_value,
            int left_cnt, int right_cnt, double left_weight, double right_weight, float gain, int missing_type, bool default_left) {
    int new_node = num_leaves - 1;
    int parent = leaf_parent[leaf];
    if (parent >= 0) {
      if (left_child[parent] == ~leaf) left_child[parent] = new_node; else right_child[parent] = new_node;
    }
    split_feature_inner[new_node] = feature;
    split_feature[new_node] = real_feature;
    split_gain[new_node] = gain;
    left_child[new_node] = ~leaf;
    right_child[new_node] = ~num_leaves;
    leaf_parent[leaf] = new_node;
    leaf_parent[num_leaves] = new_node;
    internal_weight[new_node] = leaf_weight[leaf];     // [UPSTREAM 3.2.x: parent's stored leaf weight; 0 for the root]
    internal_value[new_node] = leaf_value[leaf];
    internal_count[new_node] = left_cnt + right_cnt;
    leaf_value[leaf] = std::isnan(left_value) ? 0.0 : left_value;
    leaf_weight[leaf] = left_weight;
    leaf_count[leaf] = left_cnt;
    leaf_value[num_leaves] = std::isnan(right_value) ? 0.0 : right_value;
    leaf_weight[num_leaves] = right_weight;
    leaf_count[num_leaves] = right_cnt;
    leaf_depth[num_leaves] = leaf_depth[leaf] + 1;
    leaf_depth[leaf]++;
    decision_type[new_node] = 0;
    if (default_left) decision_type[new_node] |= 2;
    decision_type[new_node] = static_cast<int8_t>((decision_type[new_node] & 3) | (missing_type << 2));
    threshold_in_bin[new_node] = thr_bin;
    threshold[new_node] = AvoidInf(thr_double);
    ++num_leaves;
    return num_leaves - 1;
  }
  int SplitCategorical(int leaf, int feature, int real_feature, const std::vector<uint32_t>& bits_inner, const std::vector<uint32_t>& bits,
                       double left_value, double right_value, int left_cnt, int right_cnt, double left_weight, double right_weight, float gain,
                       int missing_type) {
    int new_leaf = Split(leaf, feature, real_feature, 0, 0.0, left_value, right_value, left_cnt, right_cnt, left_weight, right_weight, gain, missing_type, false);
    int node = num_leaves - 2;
    decision_type[node] = static_cast<int8_t>(1 | (missing_type << 2));
    threshold_in_bin[node] = num_cat;
    threshold[node] = num_cat;
    ++num_cat;
    cat_boundaries.push_back(cat_boundaries.back() + static_cast<int>(bits.size()));
    cat_threshold.insert(cat_threshold.end(), bits.begin(), bits.end());
    cat_boundaries_inner.push_back(cat_boundaries_inner.back() + static_cast<int>(bits_inner.size()));
    cat_threshold_inner.insert(cat_threshold_inner.end(), bits_inner.begin(), bits_inner.end());
    return new_leaf;
  }
  // traversal on BINNED data (how LightGBM ScoreUpdater::AddScore(tree, cur_tree_id) scores out-of-bag rows): numerical bin <= threshold_in_bin, NaN bin by default_left,
  // categorical by the inner (bin) bitset
  template <typename GetBin>
  int LeafByBins(GetBin bin_of, const std::vector<int>& nan_bin_of_inner) const {
    if (num_leaves <= 1) return 0;
    int node = 0;
    while (node >= 0) {
      const int f = split_feature_inner[node];
      const uint32_t bin = bin_of(f);
      bool left;
      if (decision_type[node] & 1) {
        int ci = static_cast<int>(threshold_in_bin[node]);
        left = FindInBitset(cat_threshold_inner.data() + cat_boundaries_inner[ci], cat_boundaries_inner[ci + 1] - cat_boundaries_inner[ci], static_cast<int>(bin));
      } else if (((decision_type[node] >> 2) & 3) == kMissNaN && static_cast<int>(bin) == nan_bin_of_inner[f]) left = decision_type[node] & 2;
      else left = bin <= threshold_in_bin[node];
      node = left ? left_child[node] : right_child[node];
    }
    return ~node;
  }
  void Shrinkage(double rate) {
    for (int i = 0; i < num_leaves - 1; ++i) { leaf_value[i] = MaybeRoundToZero(leaf_value[i] * rate); internal_value[i] = MaybeRoundToZero(internal_value[i] * rate); }
    leaf_value[num_leaves - 1] = MaybeRoundToZero(leaf_value[num_leaves - 1] * rate);
    shrinkage *= rate;
  }
  void AddBias(double val) {
    for (int i = 0; i < num_leaves - 1; ++i) { leaf_value[i] = MaybeRoundToZero(leaf_value[i] + val); internal_value[i] = MaybeRoundToZero(internal_value[i] + val); }
    leaf_value[num_leaves - 1] = MaybeRoundToZero(leaf_value[num_leaves - 1] + val);
    shrinkage = 1.0;
  }
  void AsConstantTree(double val) { num_leaves = 1; shrinkage = 1.0; leaf_value[0] = val; }
  double Predict(const double* row) const {
    if (num_leaves <= 1) return leaf_value[0];
    int node = 0;
    while (node >= 0) {
      double fval = row[split_feature[node]];
      int mt = (decision_type[node] >> 2) & 3;
      if (decision_type[node] & 1) {     // CategoricalDecision: NaN goes right whatever the missing type (int(NaN) = INT_MIN on x86)
        bool left = false;
        if (!std::isnan(fval)) {
          int iv = static_cast<int>(fval);
          if (iv >= 0) {
            int ci = static_cast<int>(threshold[node]);
            left = FindInBitset(cat_threshold.data() + cat_boundaries[ci], cat_boundaries[ci + 1] - cat_boundaries[ci], iv);
          }
        }
        node = left ? left_child[node] : right_child[node];
        continue;
      }
      if (std::isnan(fval) && mt != kMissNaN) fval = 0.0;
      bool go_left;
      if ((mt == kMissZero && std::fabs(fval) <= kZeroThreshold) || (mt == kMissNaN && std::isnan(fval))) go_left = decision_type[node] & 2;
      else go_left = fval <= threshold[node];
      node = go_left ? left_child[node] : right_child[node];
    }
    return leaf_value[~node];
  }
  template <typename T>
  static std::string Arr(const std::vector<T>& v, int n, const char* fmt) {
    std::string s;
    char buf[64];
    for (int i = 0; i < n; ++i) {
      if (i) s += ' ';
      if constexpr (std::is_floating_point<T>::value) snprintf(buf, sizeof(buf), fmt, static_cast<double>(v[i]));
      else snprintf(buf, sizeof(buf), fmt, static_cast<int>(v[i]));
      s += buf;
    }
    return s;
  }
  std::string ToString() const {
    std::ostringstream s;
    int nl = num_leaves;
    s << "num_leaves=" << nl << '\n';
    s << "num_cat=" << num_cat << '\n';
    s << "split_feature=" << Arr(split_feature, nl - 1, "%d") << '\n';
    s << "split_gain=" << Arr(split_gain, nl - 1, "%g") << '\n';
    s << "threshold=" << Arr(threshold, nl - 1, "%.17g") << '\n';
    s << "decision_type=" << Arr(decision_type, nl - 1, "%d") << '\n';
    s << "left_child=" << Arr(left_child, nl - 1, "%d") << '\n';
    s << "right_child=" << Arr(right_child, nl - 1, "%d") << '\n';
    s << "leaf_value=" << Arr(leaf_value, nl, "%.17g") << '\n';
    s << "leaf_weight=" << Arr(leaf_weight, nl, "%.17g") << '\n';
    s << "leaf_count=" << Arr(leaf_count, nl, "%d") << '\n';
    s << "internal_value=" << Arr(internal_value, nl - 1, "%g") << '\n';
    s << "internal_weight=" << Arr(internal_weight, nl - 1, "%g") << '\n';
    s << "internal_count=" << Arr(internal_count, nl - 1, "%d") << '\n';
    if (num_cat > 0) {
      s << "cat_boundaries=" << Arr(cat_boundaries, num_cat + 1, "%d") << '\n';
      std::string ct;
      for (size_t i = 0; i < cat_threshold.size(); ++i) ct += (i ? " " : "") + std::to_string(cat_threshold[i]);
      s << "cat_threshold=" << ct << '\n';
    }
    s << "is_linear=0\n";
    char buf[64];
    snprintf(buf, sizeof(buf), "%g", shrinkage);
    s << "shrinkage=" << buf << '\n';
    s << '\n';
    return s.str();
  }
};

// ------------------------------------------------------------------ trace (the parity artefact)
struct SplitRec {
  int tree, split, leaf, feature, threshold_bin, left_count, right_count, default_left;
  double gain, left_sum_g, left_sum_h, right_sum_g, right_sum_h, left_out, right_out;
  int smaller_rows;     // rows the histogram pass scanned for this split's children decision (local rows of the built leaf)
  int pad;
};

// ------------------------------------------------------------------ tree learner
// [UPSTREAM treelearner/serial_tree_learner.cpp + data_parallel_tree_learner.cpp]
// `parallel` (num_ranks > 1) emulates the data-parallel learner: histograms are global sums, the
// leaf counts used for gating / smaller-leaf choice / recorded in the tree are the hessian-
// reconstructed global counts carried by SplitInfo (SURVEY.md A.6, R4).
struct TreeLearner {
  const Dataset* ds = nullptr;
  Config cfg;
  SplitCfg sc;
  bool parallel = false;
  int nf = 0;
  std::vector<int> idx, tmp_left, tmp_right;          // data partition
  std::vector<int> leaf_begin, leaf_cnt;
  std::vector<int> global_cnt;                         // counts used for decisions
  std::vector<std::vector<double>> pool;               // per-leaf hist: feature u at hoff[u], max(256, num_bin) (g,h) pairs
  std::vector<size_t> hoff;                            // [nf+1] offsets in doubles
  std::vector<std::vector<uint8_t>> splittable;        // per-leaf per-feature flag
  std::vector<SplitInfo> best;
  std::vector<double> leaf_sum_g, leaf_sum_h;
  std::vector<float> og, oh;                           // ordered gradients
  std::vector<SplitRec>* trace = nullptr;
  int cur_tree = 0;
  std::vector<uint8_t> feature_used;                   // ColSampler::is_feature_used_ (by tree)
  Random col_rand{2};
  double hist_seconds = 0;
  long long hist_cells = 0;

  void Init(const Dataset* d, const Config& c, bool par) {
    ds = d; cfg = c; parallel = par;
    nf = static_cast<int>(d->used.size());
    hoff.assign(nf + 1, 0);
    for (int u = 0; u < nf; ++u) hoff[u + 1] = hoff[u] + 2 * static_cast<size_t>(std::max(256, d->mappers[d->used[u]].num_bin));
    sc = {c.lambda_l1, c.lambda_l2, c.max_delta_step, c.min_gain_to_split, c.min_sum_hessian_in_leaf, c.min_data_in_leaf};
    sc.max_cat_threshold = c.max_cat_threshold; sc.max_cat_to_onehot = c.max_cat_to_onehot; sc.min_data_per_group = c.min_data_per_group;
    sc.cat_l2 = c.cat_l2; sc.cat_smooth = c.cat_smooth;
    idx.resize(d->n); tmp_left.resize(d->n); tmp_right.resize(d->n); og.resize(d->n); oh.resize(d->n);
    int L = c.num_leaves;
    leaf_begin.assign(L, 0); leaf_cnt.assign(L, 0); global_cnt.assign(L, 0);
    pool.assign(L, std::vector<double>());
    splittable.assign(L, std::vector<uint8_t>());
    best.assign(L, SplitInfo());
    leaf_sum_g.assign(L, 0); leaf_sum_h.assign(L, 0);
    col_rand = Random(c.feature_fraction_seed);
    feature_used.assign(nf, 1);
    ResetByTree();    // [UPSTREAM ColSampler::SetTrainingData draws once at init, then once per tree]
  }
  void ResetByTree() {
    if (cfg.feature_fraction >= 1.0) return;
    int total = nf;
    int cnt = std::max(RoundInt(total * cfg.feature_fraction), std::min(2, total));
    std::fill(feature_used.begin(), feature_used.end(), 0);
    for (int i : col_rand.Sample(total, cnt)) feature_used[i] = 1;
  }
  static double now() {
#ifdef _OPENMP
    return omp_get_wtime();
#else
    return 0;
#endif
  }
  void BuildHist(int leaf, const float* g, const float* h, std::vector<double>& out, const std::vector<uint8_t>& use) {
    double t0 = now();
    out.assign(hoff[nf], 0.0);
    const int b = leaf_begin[leaf], cnt = leaf_cnt[leaf];
    const int* rows = idx.data() + b;
    const bool root = (cnt == ds->n) && rows[0] == 0 && rows[cnt - 1] == cnt - 1;
    if (!root) {
#pragma omp parallel for schedule(static)
      for (int i = 0; i < cnt; ++i) { og[i] = g[rows[i]]; oh[i] = h[rows[i]]; }
    }
    const float* gg = root ? g : og.data();
    const float* hh = root ? h : oh.data();
    const int n = ds->n;
#pragma omp parallel for schedule(dynamic, 1)
    for (int u = 0; u < nf; ++u) {
      if (!use[u]) continue;
      double* o = &out[hoff[u]];
      if (ds->wide) {
        const uint16_t* col = &ds->bins16[static_cast<size_t>(u) * n];
        if (root) { for (int i = 0; i < cnt; ++i) { int ti = col[i] << 1; o[ti] += gg[i]; o[ti + 1] += hh[i]; } }
        else { for (int i = 0; i < cnt; ++i) { int ti = col[rows[i]] << 1; o[ti] += gg[i]; o[ti + 1] += hh[i]; } }
        continue;
      }
      const uint8_t* col = &ds->bins[static_cast<size_t>(u) * n];
      if (root) {
        for (int i = 0; i < cnt; ++i) { int ti = col[i] << 1; o[ti] += gg[i]; o[ti + 1] += hh[i]; }
      } else {
        for (int i = 0; i < cnt; ++i) { int ti = col[rows[i]] << 1; o[ti] += gg[i]; o[ti + 1] += hh[i]; }
      }
    }
    hist_seconds += now() - t0;
    hist_cells += static_cast<long long>(cnt) * nf;
  }
  void FindForLeaf(int leaf, const std::vector<double>& hist, int num_data) {
    std::vector<SplitInfo> cand(nf);
    std::vector<uint8_t>& flag = splittable[leaf];
#pragma omp parallel for schedule(static)
    for (int u = 0; u < nf; ++u) {
      cand[u] = SplitInfo();
      if (!flag[u]) continue;
      const BinMapper& bm = ds->mappers[ds->used[u]];
      ScanMeta m{bm.num_bin, bm.missing_type, static_cast<int>(bm.default_bin), bm.most_freq_bin == 0 ? 1 : 0};
      bool ok = false;
      if (bm.is_categorical) FindBestThresholdCategorical(&hist[hoff[u]], m, sc, leaf_sum_g[leaf], leaf_sum_h[leaf], num_data, &cand[u], &ok);
      else FindBestThresholdNumerical(&hist[hoff[u]], m, sc, leaf_sum_g[leaf], leaf_sum_h[leaf], num_data, &cand[u], &ok);
      cand[u].feature = ds->used[u];
      flag[u] = ok ? 1 : 0;
    }
    SplitInfo b;
    for (int u = 0; u < nf; ++u) if (cand[u].feature >= 0 && cand[u].better_than(b)) b = cand[u];
    best[leaf] = b;
  }
  Tree* Train(const float* g, const float* h, const std::vector<int>* bag = nullptr) {
    const int n = ds->n;
    const int L = cfg.num_leaves;
    Tree* tree = new Tree(L);
    int nroot = n;
    if (bag) { nroot = static_cast<int>(bag->size()); std::copy(bag->begin(), bag->end(), idx.begin()); }   // SetBaggingData: the root holds the in-bag rows
    else std::iota(idx.begin(), idx.end(), 0);
    leaf_begin[0] = 0; leaf_cnt[0] = nroot; global_cnt[0] = nroot;
    for (int i = 0; i < L; ++i) best[i] = SplitInfo();
    double sg = 0, sh = 0;
#pragma omp parallel for schedule(static) reduction(+ : sg, sh)
    for (int i = 0; i < nroot; ++i) { sg += g[idx[i]]; sh += h[idx[i]]; }
    leaf_sum_g[0] = sg; leaf_sum_h[0] = sh;
    ResetByTree();
    splittable[0].assign(feature_used.begin(), feature_used.end());
    int left_leaf = 0, right_leaf = -1;
    for (int split = 0; split < L - 1; ++split) {
      // BeforeFindBestSplit
      bool go = true;
      if (cfg.max_depth > 0 && tree->leaf_depth[left_leaf] >= cfg.max_depth) {
        best[left_leaf].gain = kMinScore;
        if (right_leaf >= 0) best[right_leaf].gain = kMinScore;
        go = false;
      }
      int smaller = left_leaf, larger = -1;
      if (go) {
        int nl = global_cnt[left_leaf], nr = right_leaf >= 0 ? global_cnt[right_leaf] : 0;
        if (nr < cfg.min_data_in_leaf * 2 && nl < cfg.min_data_in_leaf * 2) {
          best[left_leaf].gain = kMinScore;
          if (right_leaf >= 0) best[right_leaf].gain = kMinScore;
          go = false;
        } else if (right_leaf >= 0) {
          if (nl < nr) { smaller = left_leaf; larger = right_leaf; } else { smaller = right_leaf; larger = left_leaf; }
        }
      }
      int smaller_rows = 0;
      if (go) {
        if (larger >= 0) {
          // parent's histogram lives in slot `left_leaf`; the larger child inherits it
          if (larger != left_leaf) { pool[larger].swap(pool[left_leaf]); }
          // children inherit the parent's per-feature splittable flags
          std::vector<uint8_t> pf = splittable[left_leaf];
          if (!cfg.oracle_inherit_splittable) pf.assign(feature_used.begin(), feature_used.end());
          splittable[left_leaf] = pf; splittable[right_leaf] = pf;
        }
        smaller_rows = leaf_cnt[smaller];
        BuildHist(smaller, g, h, pool[smaller], splittable[smaller]);
        FindForLeaf(smaller, pool[smaller], global_cnt[smaller]);
        if (larger >= 0) {
          std::vector<double>& ph = pool[larger];
          const std::vector<double>& shist = pool[smaller];
#pragma omp parallel for schedule(static)
          for (int u = 0; u < nf; ++u) {
            if (!splittable[larger][u]) continue;
            for (size_t k = hoff[u]; k < hoff[u + 1]; ++k) ph[k] -= shist[k];
          }
          FindForLeaf(larger, ph, global_cnt[larger]);
        }
      }
      // ArgMax over leaves with SplitInfo::operator>
      int best_leaf = 0;
      for (int i = 1; i < tree->num_leaves; ++i) if (best[i].better_than(best[best_leaf])) best_leaf = i;
      SplitInfo& bs = best[best_leaf];
      if (bs.gain <= 0.0) break;
      // Split
      const int inner = ds->inner_of[bs.feature];
      const BinMapper& bm = ds->mappers[bs.feature];
      int b0 = leaf_begin[best_leaf], c0 = leaf_cnt[best_leaf];
      int nl = 0, nr = 0;
      std::vector<uint32_t> bits_inner;
      if (bm.is_categorical) { std::vector<int> v(bs.cat_threshold.begin(), bs.cat_threshold.end()); bits_inner = ConstructBitset(v); }
      for (int i = 0; i < c0; ++i) {
        int r = idx[b0 + i];
        uint32_t bin = ds->bin_at(static_cast<size_t>(inner), static_cast<size_t>(r));
        bool left;
        if (bm.is_categorical) left = FindInBitset(bits_inner.data(), static_cast<int>(bits_inner.size()), static_cast<int>(bin));
        else if (bm.missing_type == kMissNaN && bin == static_cast<uint32_t>(bm.num_bin - 1)) left = bs.default_left;
        else if (bm.missing_type == kMissZero && bin == bm.default_bin) left = bs.default_left;
        else left = bin <= bs.threshold;
        if (left) tmp_left[nl++] = r; else tmp_right[nr++] = r;
      }
      std::copy(tmp_left.begin(), tmp_left.begin() + nl, idx.begin() + b0);
      std::copy(tmp_right.begin(), tmp_right.begin() + nr, idx.begin() + b0 + nl);
      int new_leaf = tree->num_leaves;
      leaf_cnt[best_leaf] = nl; leaf_begin[new_leaf] = b0 + nl; leaf_cnt[new_leaf] = nr;
      if (!parallel) { bs.left_count = nl; bs.right_count = nr; }   // update_cnt only in the serial learner
      if (trace) {
        SplitRec r{cur_tree, split, best_leaf, bs.feature, static_cast<int>(bs.threshold), bs.left_count, bs.right_count, bs.default_left,
                   bs.gain, bs.left_sum_gradient, bs.left_sum_hessian, bs.right_sum_gradient, bs.right_sum_hessian, bs.left_output,
                   bs.right_output, smaller_rows, 0};
        trace->push_back(r);
      }
      if (bm.is_categorical) {
        std::vector<int> cats;
        for (uint32_t b : bs.cat_threshold) cats.push_back(bm.bin_2_cat[b]);
        tree->SplitCategorical(best_leaf, inner, bs.feature, bits_inner, ConstructBitset(cats), bs.left_output, bs.right_output, bs.left_count,
                               bs.right_count, bs.left_sum_hessian, bs.right_sum_hessian, static_cast<float>(bs.gain + cfg.min_gain_to_split),
                               bm.missing_type);
      } else
      tree->Split(best_leaf, inner, bs.feature, bs.threshold, bm.upper[bs.threshold], bs.left_output, bs.right_output, bs.left_count,
                  bs.right_count, bs.left_sum_hessian, bs.right_sum_hessian, static_cast<float>(bs.gain + cfg.min_gain_to_split),
                  bm.missing_type, bs.default_left);
      left_leaf = best_leaf; right_leaf = new_leaf;
      global_cnt[left_leaf] = bs.left_count; global_cnt[right_leaf] = bs.right_count;
      leaf_sum_g[left_leaf] = bs.left_sum_gradient; leaf_sum_h[left_leaf] = bs.left_sum_hessian;
      leaf_sum_g[right_leaf] = bs.right_sum_gradient; leaf_sum_h[right_leaf] = bs.right_sum_hessian;
      // note: upstream decides smaller/larger for the next round inside BeforeFindBestSplit from the
      // (global) counts — done at the top of the loop.
      best[left_leaf].gain = kMinScore; best[right_leaf] = SplitInfo();
      best[left_leaf] = SplitInfo();
    }
    return tree;
  }
};

// ------------------------------------------------------------------ GBDT [UPSTREAM boosting/gbdt.cpp]
struct Booster {
  Dataset* ds = nullptr;
  Config cfg;
  std::unique_ptr<Objective> obj;
  TreeLearner learner;
  std::vector<std::unique_ptr<Tree>> models;
  std::vector<double> score;       // [K][n]
  std::vector<float> grad, hess;
  std::vector<SplitRec> trace;
  std::vector<bool> class_need_train;
  int K = 1, iter = 0, num_ranks = 1;
  bool has_init_score = false;
  double shrinkage_rate = 0.1;
  std::string model_str;
  // bagging / GOSS / RF  [LightGBM src/boosting/gbdt.cpp Bagging/BaggingHelper, goss.hpp, rf.hpp]
  std::vector<Random> bagging_rands;        // one LCG per 1024-row block of every rank's shard
  std::vector<int> block_of_row_base;       // per rank: first block index
  std::vector<int> bag_idx;
  bool balanced_bagging = false, use_bag = false, need_re_bagging = false, is_rf = false, is_goss = false, average_output = false;
  std::vector<double> rf_init_scores;
  std::vector<int> nan_bin_of_inner;
  // DART [LightGBM src/boosting/dart.hpp]
  bool is_dart = false;
  Random random_for_drop{4};
  std::vector<int> drop_index;
  std::vector<double> tree_weight;
  double sum_weight = 0.0;

  void Init(Dataset* d, const char* params) {
    ds = d;
    cfg.parse(params);
    num_ranks = static_cast<int>(d->rank_rows.size());
    obj.reset(CreateObjective(cfg));
    if (!obj) return;
    obj->Init(d, cfg);
    K = obj->num_tree_per_iter;
    shrinkage_rate = cfg.learning_rate;
    learner.Init(d, cfg, num_ranks > 1);
    learner.trace = &trace;
    score.assign(static_cast<size_t>(K) * d->n, 0.0);
    if (!d->init_score.empty()) {
      has_init_score = true;
      for (size_t i = 0; i < score.size() && i < d->init_score.size(); ++i) score[i] = d->init_score[i];
    }
    grad.resize(score.size()); hess.resize(score.size());
    class_need_train.assign(K, true);
    for (int k = 0; k < K; ++k) class_need_train[k] = obj->ClassNeedTrain(k);
    for (int f : d->used) nan_bin_of_inner.push_back(d->mappers[f].missing_type == kMissNaN && !d->mappers[f].is_categorical ? d->mappers[f].num_bin - 1 : -1);
    is_rf = cfg.boosting == "rf"; is_goss = cfg.boosting == "goss"; is_dart = cfg.boosting == "dart";
    random_for_drop = Random(cfg.drop_seed);
    // [LightGBM GBDT::ResetBaggingConfig] balanced bagging needs positive rows, i.e. the binary objective
    balanced_bagging = (cfg.pos_bagging_fraction < 1.0 || cfg.neg_bagging_fraction < 1.0) && cfg.objective == "binary" && cfg.bagging_freq > 0 &&
                       std::any_of(d->label.begin(), d->label.end(), [](float v) { return v > 0; });
    const bool bagging = (cfg.bagging_fraction < 1.0 || balanced_bagging) && cfg.bagging_freq > 0;
    if (bagging || is_goss) {
      int blocks = 0;
      for (int r = 0; r < num_ranks; ++r) {
        block_of_row_base.push_back(blocks);
        int nb = (d->rank_rows[r] + 1023) / 1024;
        for (int i = 0; i < nb; ++i) bagging_rands.emplace_back(cfg.bagging_seed + i);     // every rank seeds its own blocks from bagging_seed
        blocks += nb;
      }
      need_re_bagging = bagging;
    }
    if (is_rf) {
      average_output = true;
      shrinkage_rate = 1.0;
      rf_init_scores.assign(K, 0.0);
      for (int k = 0; k < K; ++k) rf_init_scores[k] = InitScoreValue(k);
      std::vector<double> tmp(score.size());
      for (int k = 0; k < K; ++k) std::fill(tmp.begin() + static_cast<size_t>(k) * d->n, tmp.begin() + static_cast<size_t>(k + 1) * d->n, rf_init_scores[k]);
      obj->GetGradients(tmp.data(), grad.data(), hess.data());      // "only boosting one time"
    }
  }
  double InitScoreValue(int k) {       // BoostFromAverage(k, update_scorer = false)
    if (models.empty() && !has_init_score && cfg.boost_from_average) {
      double init;
      if (num_ranks == 1 || obj->GlobalInitScore()) init = obj->BoostFromScore(k, 0, ds->n);
      else { double s = 0; int off = 0; for (int r = 0; r < num_ranks; ++r) { s += obj->BoostFromScore(k, off, off + ds->rank_rows[r]); off += ds->rank_rows[r]; } init = s / num_ranks; }
      if (std::fabs(init) > kEpsilon) return init;
    }
    return 0.0;
  }
  void Bagging(int it) {
    const int n = ds->n;
    if (is_goss) {
      use_bag = false;
      if (it < static_cast<int>(1.0f / cfg.learning_rate)) return;      // no subsampling for the first 1/lr iterations
      bag_idx.clear();
      int off = 0;
      for (int r = 0; r < num_ranks; ++r) {
        const int ln = ds->rank_rows[r];
        for (int c0 = 0; c0 < ln; c0 += 1024) {          // one chunk per 1024-row block (LightGBM chunks by thread count; this equals it when num_threads >= n/1024)
          const int cnt = std::min(1024, ln - c0);
          Random& rnd = bagging_rands[block_of_row_base[r] + c0 / 1024];
          std::vector<float> tg(cnt, 0.0f);
          for (int i = 0; i < cnt; ++i)
            for (int k = 0; k < K; ++k) { size_t id = static_cast<size_t>(k) * n + off + c0 + i; tg[i] += std::fabs(grad[id] * hess[id]); }
          int top_k = std::max(1, static_cast<int>(cnt * cfg.top_rate));
          int other_k = static_cast<int>(cnt * cfg.other_rate);
          std::vector<float> sorted(tg);
          std::nth_element(sorted.begin(), sorted.begin() + top_k - 1, sorted.end(), std::greater<float>());
          const float threshold = sorted[top_k - 1];
          const float multiply = static_cast<float>(cnt - top_k) / other_k;
          int left = 0, big = 0;
          for (int i = 0; i < cnt; ++i) {
            if (tg[i] >= threshold) { bag_idx.push_back(off + c0 + i); ++left; ++big; }
            else {
              int sampled = left - big, rest_need = other_k - sampled, rest_all = (cnt - i) - (top_k - big);
              double prob = rest_need / static_cast<double>(rest_all);
              if (rnd.NextFloat() < prob) {
                bag_idx.push_back(off + c0 + i); ++left;
                for (int k = 0; k < K; ++k) { size_t id = static_cast<size_t>(k) * n + off + c0 + i; grad[id] *= multiply; hess[id] *= multiply; }
              }
            }
          }
        }
        off += ln;
      }
      use_bag = true;
      return;
    }
    const bool bagging = (cfg.bagging_fraction < 1.0 || balanced_bagging) && cfg.bagging_freq > 0;
    if (!bagging) return;
    if ((use_bag && it % cfg.bagging_freq == 0) || need_re_bagging) {
      need_re_bagging = false;
      bag_idx.clear();
      int off = 0;
      for (int r = 0; r < num_ranks; ++r) {
        for (int i = 0; i < ds->rank_rows[r]; ++i)
          if (bagging_rands[block_of_row_base[r] + i / 1024].NextFloat() <
              (balanced_bagging ? (ds->label[off + i] > 0 ? cfg.pos_bagging_fraction : cfg.neg_bagging_fraction) : cfg.bagging_fraction))
            bag_idx.push_back(off + i);
        off += ds->rank_rows[r];
      }
      use_bag = true;
    }
  }
  // ScoreUpdater::AddScore(tree, cur_tree_id) for an arbitrary stored tree: every row walks the tree on its bins
  void AddStoredTree(const Tree& t, int k) {
    const int n = ds->n;
    double* sp = &score[static_cast<size_t>(k) * n];
    if (t.num_leaves <= 1) { if (t.leaf_value[0] != 0.0) for (int i = 0; i < n; ++i) sp[i] += t.leaf_value[0]; return; }
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
      int leaf = t.LeafByBins([&](int f) { return ds->bin_at(static_cast<size_t>(f), static_cast<size_t>(i)); }, nan_bin_of_inner);
      sp[i] += t.leaf_value[leaf];
    }
  }
  void DroppingTrees() {       // DART::DroppingTrees
    drop_index.clear();
    bool is_skip = random_for_drop.NextFloat() < cfg.skip_drop;
    if (!is_skip) {
      double drop_rate = cfg.drop_rate;
      if (!cfg.uniform_drop) {
        double inv_average_weight = static_cast<double>(tree_weight.size()) / sum_weight;
        if (cfg.max_drop > 0) drop_rate = std::min(drop_rate, cfg.max_drop * inv_average_weight / sum_weight);
        for (int i = 0; i < iter; ++i)
          if (random_for_drop.NextFloat() < drop_rate * tree_weight[i] * inv_average_weight) {
            drop_index.push_back(i);
            if (drop_index.size() >= static_cast<size_t>(cfg.max_drop)) break;
          }
      } else {
        if (cfg.max_drop > 0) drop_rate = std::min(drop_rate, cfg.max_drop / static_cast<double>(iter));
        for (int i = 0; i < iter; ++i)
          if (random_for_drop.NextFloat() < drop_rate) {
            drop_index.push_back(i);
            if (drop_index.size() >= static_cast<size_t>(cfg.max_drop)) break;
          }
      }
    }
    for (int i : drop_index)
      for (int k = 0; k < K; ++k) { Tree& t = *models[static_cast<size_t>(i) * K + k]; t.Shrinkage(-1.0); AddStoredTree(t, k); }
    if (!cfg.xgboost_dart_mode) shrinkage_rate = cfg.learning_rate / (1.0f + static_cast<double>(drop_index.size()));
    else if (drop_index.empty()) shrinkage_rate = cfg.learning_rate;
    else shrinkage_rate = cfg.learning_rate / (cfg.learning_rate + static_cast<double>(drop_index.size()));
  }
  void Normalize() {           // DART::Normalize (train scores only; the oracle holds no validation sets)
    const double k = static_cast<double>(drop_index.size());
    for (int i : drop_index) {
      for (int c = 0; c < K; ++c) {
        Tree& t = *models[static_cast<size_t>(i) * K + c];
        if (!cfg.xgboost_dart_mode) { t.Shrinkage(1.0f / (k + 1.0f)); t.Shrinkage(-k); }
        else { t.Shrinkage(shrinkage_rate); t.Shrinkage(-k / cfg.learning_rate); }
        AddStoredTree(t, c);
      }
      if (!cfg.uniform_drop) {
        if (!cfg.xgboost_dart_mode) { sum_weight -= tree_weight[i] * (1.0f / (k + 1.0f)); tree_weight[i] *= (k / (k + 1.0f)); }
        else { sum_weight -= tree_weight[i] * (1.0f / (k + cfg.learning_rate)); tree_weight[i] *= (k / (k + cfg.learning_rate)); }
      }
    }
  }
  // SerialTreeLearner::RenewTreeOutput: every leaf's output is re-fitted on the residuals of its (in-bag) rows; with several
  // ranks each fits its own shard's rows and the outputs are averaged over the ranks that hold rows of the leaf
  void RenewTreeOutput(Tree* t, const std::function<double(int)>& residual) {
    if (!obj->IsRenewTreeOutput()) return;
    std::vector<int> rank_end;
    { int off = 0; for (int r = 0; r < num_ranks; ++r) { off += ds->rank_rows[r]; rank_end.push_back(off); } }
    for (int l = 0; l < t->num_leaves; ++l) {
      const int b = learner.leaf_begin[l], c = learner.leaf_cnt[l];
      double sum = 0.0; int workers = 0;
      int i = 0;
      for (int r = 0; r < num_ranks; ++r) {
        std::vector<int> rows;
        while (i < c && learner.idx[b + i] < rank_end[r]) rows.push_back(learner.idx[b + i++]);
        if (!rows.empty()) { sum += obj->RenewTreeOutput(rows, residual); ++workers; }
      }
      t->leaf_value[l] = num_ranks > 1 ? sum / workers : sum;
    }
  }
  void AddTreeToScores(const Tree& t, int k) {        // UpdateScore: in-bag via the partition, out-of-bag by binned traversal == tree(row) for all rows
    const int n = ds->n;
    double* sp = &score[static_cast<size_t>(k) * n];
    if (!use_bag) {
      for (int l = 0; l < t.num_leaves; ++l) {
        double v = t.leaf_value[l];
        int b = learner.leaf_begin[l], c = learner.leaf_cnt[l];
        for (int i = 0; i < c; ++i) sp[learner.idx[b + i]] += v;
      }
      return;
    }
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
      int leaf = t.LeafByBins([&](int f) { return ds->bin_at(static_cast<size_t>(f), static_cast<size_t>(i)); }, nan_bin_of_inner);
      sp[i] += t.leaf_value[leaf];
    }
  }
  double BoostFromAverage(int k) {
    if (models.empty() && !has_init_score && cfg.boost_from_average) {
      double init;
      if (num_ranks == 1 || obj->GlobalInitScore()) init = obj->BoostFromScore(k, 0, ds->n);
      else {   // Network::GlobalSyncUpByMean of the per-rank values (SURVEY.md A.8 / R11)
        double s = 0; int off = 0;
        for (int r = 0; r < num_ranks; ++r) { s += obj->BoostFromScore(k, off, off + ds->rank_rows[r]); off += ds->rank_rows[r]; }
        init = s / num_ranks;
      }
      if (std::fabs(init) > kEpsilon) {
        double* sp = &score[static_cast<size_t>(k) * ds->n];
        for (int i = 0; i < ds->n; ++i) sp[i] += init;
        return init;
      }
    }
    return 0.0;
  }
  bool TrainOneIter() {
    const int n = ds->n;
    std::vector<double> init_scores(K, 0.0);
    if (is_rf) {
      init_scores = rf_init_scores;
    } else {
      for (int k = 0; k < K; ++k) init_scores[k] = BoostFromAverage(k);
      if (is_dart) DroppingTrees();        // GetTrainingScore() inside Boosting(): drop before the gradients are taken
      obj->GetGradients(score.data(), grad.data(), hess.data());
    }
    Bagging(iter);
    bool should_continue = false;
    for (int k = 0; k < K; ++k) {
      std::unique_ptr<Tree> t(new Tree(2));
      if (class_need_train[k] && !ds->used.empty()) {
        learner.cur_tree = static_cast<int>(models.size());
        t.reset(learner.Train(&grad[static_cast<size_t>(k) * n], &hess[static_cast<size_t>(k) * n], use_bag ? &bag_idx : nullptr));
      }
      double* sp = &score[static_cast<size_t>(k) * n];
      if (is_rf) {
        const double m0 = static_cast<double>(iter), m1 = 1.0 / (iter + 1);
        if (t->num_leaves > 1) {
          { const double pred = init_scores[k]; const float* y = ds->label.data(); RenewTreeOutput(t.get(), [=](int i) { return static_cast<double>(y[i]) - pred; }); }
          if (std::fabs(init_scores[k]) > kEpsilon) t->AddBias(init_scores[k]);
          for (int i = 0; i < n; ++i) sp[i] *= m0;
          AddTreeToScores(*t, k);
          for (int i = 0; i < n; ++i) sp[i] *= m1;
        } else if (models.size() < static_cast<size_t>(K)) {
          double output = class_need_train[k] ? init_scores[k] : obj->BoostFromScore(k, 0, n);
          t->AsConstantTree(output);
          for (int i = 0; i < n; ++i) sp[i] = (sp[i] * m0 + output) * m1;
        }
        models.push_back(std::move(t));
        continue;
      }
      if (t->num_leaves > 1) {
        should_continue = true;
        { const float* y = ds->label.data(); RenewTreeOutput(t.get(), [=](int i) { return static_cast<double>(y[i]) - sp[i]; }); }
        t->Shrinkage(shrinkage_rate);
        AddTreeToScores(*t, k);
        if (std::fabs(init_scores[k]) > kEpsilon) t->AddBias(init_scores[k]);
      } else if (models.size() < static_cast<size_t>(K)) {
        double output = class_need_train[k] ? init_scores[k] : obj->BoostFromScore(k, 0, n);
        t->AsConstantTree(output);
        for (int i = 0; i < n; ++i) sp[i] += output;
      }
      models.push_back(std::move(t));
    }
    if (is_rf) { ++iter; return false; }
    if (!should_continue) {
      if (models.size() > static_cast<size_t>(K)) for (int k = 0; k < K; ++k) models.pop_back();
      return true;
    }
    ++iter;
    if (is_dart) {
      Normalize();
      if (!cfg.uniform_drop) { tree_weight.push_back(shrinkage_rate); sum_weight += shrinkage_rate; }
    }
    return false;
  }
  std::string ModelToString() const {
    std::ostringstream ss;
    ss << "tree\n" << "version=v3\n";
    ss << "num_class=" << ((cfg.objective == "multiclass" || cfg.objective == "multiclassova") ? cfg.num_class : 1) << '\n';
    ss << "num_tree_per_iteration=" << K << '\n';
    ss << "label_index=0\n";
    ss << "max_feature_idx=" << ds->F - 1 << '\n';
    ss << "objective=" << obj->ToString() << '\n';
    if (average_output) ss << "average_output\n";
    ss << "feature_names=";
    for (int f = 0; f < ds->F; ++f) ss << (f ? " " : "") << ds->feature_names[f];
    ss << '\n' << "feature_infos=";
    for (int f = 0; f < ds->F; ++f) ss << (f ? " " : "") << ds->mappers[f].info_string();
    ss << '\n';
    std::vector<std::string> ts(models.size());
    ss << "tree_sizes=";
    for (size_t i = 0; i < models.size(); ++i) {
      ts[i] = "Tree=" + std::to_string(i) + "\n" + models[i]->ToString() + "\n";
      ss << (i ? " " : "") << ts[i].size();
    }
    ss << "\n\n";
    for (auto& s : ts) ss << s;
    ss << "end of trees\n";
    std::vector<size_t> imp(ds->F, 0);
    for (auto& m : models) for (int i = 0; i < m->num_leaves - 1; ++i) if (m->split_gain[i] > 0) imp[m->split_feature[i]]++;
    std::vector<std::pair<size_t, std::string>> pairs;
    for (int f = 0; f < ds->F; ++f) if (imp[f] > 0) pairs.emplace_back(imp[f], ds->feature_names[f]);
    std::stable_sort(pairs.begin(), pairs.end(), [](auto& a, auto& b) { return a.first > b.first; });
    ss << "\nfeature_importances:\n";
    for (auto& p : pairs) ss << p.second << "=" << p.first << '\n';
    return ss.str();
  }
};

}  // namespace orc

// ==================================================================== C interface (ctypes)
using namespace orc;
extern "C" {

void* orc_dataset_create(const double* X, int n, int F, const char* params, int num_ranks, const int* rank_rows) {
  Dataset* d = new Dataset();
  int one = n;
  if (num_ranks <= 1 || !rank_rows) { num_ranks = 1; rank_rows = &one; }
  d->build(X, n, F, params, num_ranks, rank_rows);
  return d;
}
void orc_dataset_free(void* h) { delete static_cast<Dataset*>(h); }
// Dataset from PRE-COMPUTED bins (row-major uint8 [n][F]) plus the mapper descriptions of every feature: for the mid-scale parity
// tests, where the raw matrix only ever exists on the device (synthesised in chunks) and the bins are downloaded from the product
// after they were checked row-sample-wise.  meta5[f] = {num_bin, missing_type, default_bin, most_freq_bin, is_trivial};
// upper = concatenated bin upper bounds, upper_off[F+1]; minmax[2f..2f+1] = the feature's sampled value range (feature_infos).
void* orc_dataset_create_from_bins(const uint8_t* bins_rm, int n, int F, const int* meta5, const double* upper, const int* upper_off,
                                   const double* minmax, const char* params, int num_ranks, const int* rank_rows) {
  Dataset* d = new Dataset();
  d->n = n; d->F = F;
  d->cfg.parse(params);
  int one = n;
  if (num_ranks <= 1 || !rank_rows) { num_ranks = 1; rank_rows = &one; }
  d->rank_rows.assign(rank_rows, rank_rows + num_ranks);
  d->mappers.assign(F, BinMapper());
  for (int f = 0; f < F; ++f) {
    BinMapper& m = d->mappers[f];
    m.num_bin = meta5[f * 5]; m.missing_type = meta5[f * 5 + 1]; m.default_bin = meta5[f * 5 + 2]; m.most_freq_bin = meta5[f * 5 + 3];
    m.is_trivial = meta5[f * 5 + 4] != 0;
    m.upper.assign(upper + upper_off[f], upper + upper_off[f + 1]);
    m.min_val = minmax[2 * f]; m.max_val = minmax[2 * f + 1];
  }
  d->inner_of.assign(F, -1);
  for (int f = 0; f < F; ++f) if (!d->mappers[f].is_trivial) { d->inner_of[f] = static_cast<int>(d->used.size()); d->used.push_back(f); }
  d->alloc_bins();
#pragma omp parallel for schedule(static)
  for (int u = 0; u < static_cast<int>(d->used.size()); ++u) {
    const int f = d->used[u];
    uint8_t* col = &d->bins[static_cast<size_t>(u) * n];
    for (int i = 0; i < n; ++i) col[i] = bins_rm[static_cast<size_t>(i) * F + f];
  }
  d->feature_names.resize(F);
  for (int f = 0; f < F; ++f) d->feature_names[f] = "Column_" + std::to_string(f);
  return d;
}

int orc_dataset_num_used(void* h) { return static_cast<int>(static_cast<Dataset*>(h)->used.size()); }
// bins out: row-major uint8 [n][F]; trivial features are written as 0 (bins above 255 are truncated: use orc_dataset_bins16 for wide datasets)
void orc_dataset_bins(void* h, uint8_t* out) {
  Dataset* d = static_cast<Dataset*>(h);
  std::memset(out, 0, static_cast<size_t>(d->n) * d->F);
  for (size_t u = 0; u < d->used.size(); ++u) {
    int f = d->used[u];
    for (int i = 0; i < d->n; ++i) out[static_cast<size_t>(i) * d->F + f] = static_cast<uint8_t>(d->bin_at(u, i));
  }
}
void orc_dataset_bins16(void* h, uint16_t* out) {
  Dataset* d = static_cast<Dataset*>(h);
  std::memset(out, 0, static_cast<size_t>(d->n) * d->F * sizeof(uint16_t));
  for (size_t u = 0; u < d->used.size(); ++u) {
    int f = d->used[u];
    for (int i = 0; i < d->n; ++i) out[static_cast<size_t>(i) * d->F + f] = static_cast<uint16_t>(d->bin_at(u, i));
  }
}
// categorical feature: bin -> category value (bin 0 = -1); returns num_bin
int orc_dataset_bin_to_cat(void* h, int f, int* out) {
  const BinMapper& m = static_cast<Dataset*>(h)->mappers[f];
  for (size_t i = 0; i < m.bin_2_cat.size(); ++i) out[i] = m.bin_2_cat[i];
  return static_cast<int>(m.bin_2_cat.size());
}
// info: {num_bin, missing_type, default_bin, most_freq_bin, is_trivial}
void orc_dataset_feature_info(void* h, int f, int* info) {
  const BinMapper& m = static_cast<Dataset*>(h)->mappers[f];
  info[0] = m.num_bin; info[1] = m.missing_type; info[2] = m.default_bin; info[3] = m.most_freq_bin; info[4] = m.is_trivial;
}
int orc_dataset_upper_bounds(void* h, int f, double* out) {
  const BinMapper& m = static_cast<Dataset*>(h)->mappers[f];
  for (size_t i = 0; i < m.upper.size(); ++i) out[i] = m.upper[i];
  return static_cast<int>(m.upper.size());
}
int orc_dataset_set_field(void* h, const char* name, const void* data, int n) {
  Dataset* d = static_cast<Dataset*>(h);
  std::string s(name);
  if (s == "label") d->label.assign(static_cast<const float*>(data), static_cast<const float*>(data) + n);
  else if (s == "weight") d->weight.assign(static_cast<const float*>(data), static_cast<const float*>(data) + n);
  else if (s == "init_score") d->init_score.assign(static_cast<const double*>(data), static_cast<const double*>(data) + n);
  else if (s == "group") {
    const int* g = static_cast<const int*>(data);
    d->query_boundaries.assign(1, 0);
    for (int i = 0; i < n; ++i) d->query_boundaries.push_back(d->query_boundaries.back() + g[i]);
  } else return -1;
  return 0;
}
void* orc_booster_create(void* ds, const char* params) {
  Booster* b = new Booster();
  b->Init(static_cast<Dataset*>(ds), params);
  if (!b->obj) { delete b; return nullptr; }
  return b;
}
void orc_booster_free(void* h) { delete static_cast<Booster*>(h); }
int orc_booster_update(void* h) { return static_cast<Booster*>(h)->TrainOneIter() ? 1 : 0; }
void orc_booster_reset_learning_rate(void* h, double lr) {      // GBDT::ResetConfig (+ DART::ResetConfig: drop RNG and sum_weight_ restart)
  Booster* b = static_cast<Booster*>(h);
  b->cfg.learning_rate = lr;
  if (!b->is_rf) b->shrinkage_rate = lr;
  if (b->is_dart) { b->random_for_drop = Random(b->cfg.drop_seed); b->sum_weight = 0.0; }
}
int orc_booster_num_trees(void* h) { return static_cast<int>(static_cast<Booster*>(h)->models.size()); }
const char* orc_booster_model_string(void* h) {
  Booster* b = static_cast<Booster*>(h);
  b->model_str = b->ModelToString();
  return b->model_str.c_str();
}
int orc_booster_trace_len(void* h) { return static_cast<int>(static_cast<Booster*>(h)->trace.size()); }
// 18 doubles per record: tree split leaf feature thr left_cnt right_cnt default_left gain lsg lsh rsg rsh lout rout smaller_rows
void orc_booster_trace(void* h, double* out) {
  Booster* b = static_cast<Booster*>(h);
  for (size_t i = 0; i < b->trace.size(); ++i) {
    const SplitRec& r = b->trace[i];
    double* o = out + i * 16;
    o[0] = r.tree; o[1] = r.split; o[2] = r.leaf; o[3] = r.feature; o[4] = r.threshold_bin; o[5] = r.left_count; o[6] = r.right_count;
    o[7] = r.default_left; o[8] = r.gain; o[9] = r.left_sum_g; o[10] = r.left_sum_h; o[11] = r.right_sum_g; o[12] = r.right_sum_h;
    o[13] = r.left_out; o[14] = r.right_out; o[15] = r.smaller_rows;
  }
}
void orc_booster_scores(void* h, double* out) {
  Booster* b = static_cast<Booster*>(h);
  std::memcpy(out, b->score.data(), b->score.size() * sizeof(double));
}
void orc_booster_gradients(void* h, float* g, float* hs) {
  Booster* b = static_cast<Booster*>(h);
  b->obj->GetGradients(b->score.data(), b->grad.data(), b->hess.data());
  std::memcpy(g, b->grad.data(), b->grad.size() * sizeof(float));
  std::memcpy(hs, b->hess.data(), b->hess.size() * sizeof(float));
}
// raw prediction of the whole model for nrow rows (row-major f64), out [nrow][K]
void orc_booster_predict_raw(void* h, const double* X, int nrow, int F, double* out) {
  Booster* b = static_cast<Booster*>(h);
  int K = b->K;
#pragma omp parallel for schedule(static)
  for (int i = 0; i < nrow; ++i) {
    for (int k = 0; k < K; ++k) out[static_cast<size_t>(i) * K + k] = 0;
    for (size_t t = 0; t < b->models.size(); ++t) out[static_cast<size_t>(i) * K + (t % K)] += b->models[t]->Predict(X + static_cast<size_t>(i) * F);
    if (b->average_output && !b->models.empty()) for (int k = 0; k < K; ++k) out[static_cast<size_t>(i) * K + k] /= (b->models.size() / K);
  }
}
void orc_booster_hist_stats(void* h, double* seconds, long long* cells) {
  Booster* b = static_cast<Booster*>(h);
  *seconds = b->learner.hist_seconds; *cells = b->learner.hist_cells;
}
void orc_set_num_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}
int orc_num_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

// ---- kernel-level oracles used by the GPU parity tests
// fp64 histogram of rows idx[0..cnt) (or 0..cnt if idx==NULL) over row-major uint8 bins [n][F]; out [F][256][2]
void orc_histogram(const uint8_t* bins, int n, int F, const float* g, const float* h, const int* idx, int cnt, double* out) {
  (void)n;
  std::memset(out, 0, sizeof(double) * F * 512);
#pragma omp parallel for schedule(static)
  for (int f = 0; f < F; ++f) {
    double* o = out + static_cast<size_t>(f) * 512;
    for (int i = 0; i < cnt; ++i) {
      int r = idx ? idx[i] : i;
      int b = bins[static_cast<size_t>(r) * F + f];
      o[b * 2] += g[r]; o[b * 2 + 1] += h[r];
    }
  }
}
// one feature's best numerical split.  meta = {num_bin, missing_type, default_bin, most_freq_bin}
// cfgv = {l1, l2, max_delta_step, min_gain_to_split, min_sum_hessian, min_data_in_leaf}
// out = {gain, threshold, default_left, left_count, right_count, lsg, lsh, rsg, rsh, lout, rout, splittable}
void orc_best_split(const double* hist, const int* meta, const double* cfgv, double sum_g, double sum_h, int num_data, double* out) {
  ScanMeta m{meta[0], meta[1], meta[2], meta[3] == 0 ? 1 : 0};
  SplitCfg c{cfgv[0], cfgv[1], cfgv[2], cfgv[3], cfgv[4], static_cast<int>(cfgv[5])};
  SplitInfo s;
  bool ok = false;
  FindBestThresholdNumerical(hist, m, c, sum_g, sum_h, num_data, &s, &ok);
  out[0] = s.gain; out[1] = s.threshold; out[2] = s.default_left; out[3] = s.left_count; out[4] = s.right_count;
  out[5] = s.left_sum_gradient; out[6] = s.left_sum_hessian; out[7] = s.right_sum_gradient; out[8] = s.right_sum_hessian;
  out[9] = s.left_output; out[10] = s.right_output; out[11] = ok;
}
// LightGBM's LCG sampler (utils/random.h) — pinned by tests against hand-computed values
int orc_random_sample(int seed, int N, int K, int* out) {
  Random r(seed);
  auto v = r.Sample(N, K);
  for (size_t i = 0; i < v.size(); ++i) out[i] = v[i];
  return static_cast<int>(v.size());
}
// DatasetUtils.countCardinality (lightgbm/src/main/scala/.../dataset/DatasetUtils.scala:18-40): run lengths of group ids
int orc_count_cardinality(const long long* ids, int n, int* out) {
  int m = 0;
  if (n == 0) return 0;
  long long prev = ids[0];
  int run = 1;
  for (int i = 1; i < n; ++i) {
    if (ids[i] == prev) ++run; else { out[m++] = run; run = 1; prev = ids[i]; }
  }
  out[m++] = run;
  return m;
}
}
