// Parameter-string parser for the b200gbm engine.
//
// Wire format = what MMLSpark's Scala side builds: space separated `key=value`, empty values allowed,
// later keys override earlier ones.  Reference: TrainParams.toString
// (lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/params/TrainParams.scala:47-63,83-88,108-111,131-137)
// and LightGBMBase.getDatasetParams (lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/LightGBMBase.scala:265-272).
// Keys the reference never sets keep the native LightGBM 3.2.x defaults (SURVEY.md Appendix B.2).
#pragma once
#include <climits>
#include <cmath>
#include <cstdlib>
#include <map>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace b200gbm {

// LightGBM's kEpsilon (1e-15f): path smoothing is on when path_smooth exceeds it
constexpr double kPathSmoothEps = static_cast<double>(1e-15f);

struct Config {
  // --- core
  std::string objective = "regression";
  std::string boosting = "gbdt";
  std::string tree_learner = "serial";
  std::vector<std::string> metric;          // resolved metric names
  bool metric_given = false;
  int num_iterations = 100;
  double learning_rate = 0.1;
  int num_leaves = 31;
  int num_threads = 0;
  int max_depth = -1;
  int min_data_in_leaf = 20;
  double min_sum_hessian_in_leaf = 1e-3;
  double bagging_fraction = 1.0, pos_bagging_fraction = 1.0, neg_bagging_fraction = 1.0;
  int bagging_freq = 0, bagging_seed = 3;
  double feature_fraction = 1.0;
  int feature_fraction_seed = 2;
  double feature_fraction_bynode = 1.0;     // < 1: each leaf's split is chosen among a sample of the tree's features (kernels.cuh d_bynode_sample)
  bool extra_trees = false;                 // one random threshold per (leaf, feature) scan (TreeLearner, kernels.cuh K5/K6)
  int extra_seed = 6;                       // the stream of used feature i starts at extra_seed + i
  std::vector<int> monotone_constraints;    // per real feature -1, 0 or +1; non-empty: the constrained scans (TreeLearner, kernels.cuh kMono)
  std::string monotone_constraints_method = "basic";      // only "basic" trains (Booster checks at create)
  double monotone_penalty = 0.0;            // scales a monotone split's gain down near the root (kernels.cuh d_mono_penalty)
  // > kPathSmoothEps: every split gain and leaf output is smoothed toward the parent leaf's output (kernels.cuh d_smooth_output)
  double path_smooth = 0.0;
  // sets of real feature indices; a branch's split features stay inside one set (TreeLearner sets_of_, kernels.cuh d_pick_block)
  std::vector<std::vector<int>> interaction_constraints;
  std::string interaction_constraints_malformed;      // the value given when it does not parse (Booster fails at create)
  // quantised training [UPSTREAM 4.x names and defaults, from knowledge]: each tree's g and h discretised to a few integer levels
  // (kernels.cuh k_quantize_discrete) and histograms built with one packed atomic per cell (hist_kernel.cuh k4_hist_build_packed)
  bool use_quantized_grad = false;
  int num_grad_quant_bins = 4;              // B: q_g in [-floor(B/2), floor(B/2)], q_h in [-B, B]; 2..63 (Booster checks)
  bool quant_train_renew_leaf = false;      // leaf values from the true in-bag sums of g and h after growth
  bool stochastic_rounding = true;
  // LGBM_BoosterRefit: leaf = decay * leaf + (1 - decay) * refit output (refit.cu); [0, 1] is checked by the refit, not here
  double refit_decay_rate = 0.9;
  // forced splits: a JSON file of splits every tree starts with (forced_splits.h); empty for none.  Booster reads it at create and when a
  // ResetParameter gives the key
  std::string forcedsplits_filename;
  int early_stopping_round = 0;
  double max_delta_step = 0.0, lambda_l1 = 0.0, lambda_l2 = 0.0, min_gain_to_split = 0.0;
  double cat_l2 = 10.0, cat_smooth = 10.0;
  int max_cat_threshold = 32, max_cat_to_onehot = 4, min_data_per_group = 100;
  double drop_rate = 0.1, skip_drop = 0.5;
  int max_drop = 50, drop_seed = 4;
  bool xgboost_dart_mode = false, uniform_drop = false;
  double top_rate = 0.2, other_rate = 0.1;
  int top_k = 20;
  int verbosity = 1;
  // --- dataset
  int max_bin = 255;
  int min_data_in_bin = 3;
  int bin_construct_sample_cnt = 200000;
  int data_random_seed = 1;
  bool use_missing = true, zero_as_missing = false, feature_pre_filter = true, pre_partition = false;
  bool enable_bundle = true;                // exclusive feature bundling of sparse features (bundle.h)
  std::vector<int> categorical_feature;
  std::string max_bin_by_feature;
  // --- objective
  int num_class = 1;
  bool is_unbalance = false;
  double scale_pos_weight = 1.0, sigmoid = 1.0;
  bool boost_from_average = true;
  double alpha = 0.9, tweedie_variance_power = 1.5, fair_c = 1.0, poisson_max_delta_step = 0.7;
  int objective_seed = 5;                   // rank_xendcg's random states
  int lambdarank_truncation_level = 30;
  bool lambdarank_norm = true;
  std::vector<double> label_gain;
  // [UPSTREAM 4.1, from knowledge] L2 regularisation of the ranking objectives' position factors (a training set with a position field);
  // >= 0, Booster checks at create and reset
  double lambdarank_position_bias_regularization = 0.0;
  std::vector<int> eval_at;
  std::vector<double> auc_mu_weights;       // auc_mu's K x K class-pair weights, row-major; empty = 1 off the diagonal, 0 on it
  // --- predict: read from a predict call's parameter string only, never printed (the saved params block has no predict section).
  // HostModel::PredictEarlyStop decides whether they apply and checks them.
  bool pred_early_stop = false;
  int pred_early_stop_freq = 10;
  double pred_early_stop_margin = 10.0;
  // --- network
  int num_machines = 1;
  std::map<std::string, std::string> raw;

  static bool ParseBool(const std::string& v) {
    return v == "true" || v == "True" || v == "TRUE" || v == "1" || v == "+";
  }
  static const std::map<std::string, std::string>& Aliases() {
    static const std::map<std::string, std::string> a = {
        {"boosting_type", "boosting"}, {"boost", "boosting"}, {"objective_type", "objective"},
        {"app", "objective"}, {"application", "objective"}, {"num_iteration", "num_iterations"},
        {"n_iter", "num_iterations"}, {"num_tree", "num_iterations"}, {"num_trees", "num_iterations"},
        {"num_round", "num_iterations"}, {"num_rounds", "num_iterations"}, {"num_boost_round", "num_iterations"},
        {"n_estimators", "num_iterations"}, {"shrinkage_rate", "learning_rate"}, {"eta", "learning_rate"},
        {"num_leaf", "num_leaves"}, {"max_leaves", "num_leaves"}, {"max_leaf", "num_leaves"},
        {"tree", "tree_learner"}, {"tree_type", "tree_learner"}, {"tree_learner_type", "tree_learner"},
        {"num_thread", "num_threads"}, {"nthread", "num_threads"}, {"nthreads", "num_threads"}, {"n_jobs", "num_threads"},
        {"min_data_per_leaf", "min_data_in_leaf"}, {"min_data", "min_data_in_leaf"},
        {"min_child_samples", "min_data_in_leaf"}, {"min_sum_hessian_per_leaf", "min_sum_hessian_in_leaf"},
        {"min_sum_hessian", "min_sum_hessian_in_leaf"}, {"min_hessian", "min_sum_hessian_in_leaf"},
        {"min_child_weight", "min_sum_hessian_in_leaf"}, {"sub_row", "bagging_fraction"},
        {"subsample", "bagging_fraction"}, {"bagging", "bagging_fraction"}, {"subsample_freq", "bagging_freq"},
        {"bagging_fraction_seed", "bagging_seed"}, {"sub_feature", "feature_fraction"},
        {"colsample_bytree", "feature_fraction"}, {"sub_feature_bynode", "feature_fraction_bynode"},
        {"colsample_bynode", "feature_fraction_bynode"}, {"extra_tree", "extra_trees"}, {"early_stopping_rounds", "early_stopping_round"},
        {"mc", "monotone_constraints"}, {"monotone_constraint", "monotone_constraints"},
        {"monotone_constraining_method", "monotone_constraints_method"}, {"mc_method", "monotone_constraints_method"},
        {"monotone_splits_penalty", "monotone_penalty"}, {"ms_penalty", "monotone_penalty"}, {"mc_penalty", "monotone_penalty"},
        {"early_stopping", "early_stopping_round"}, {"n_iter_no_change", "early_stopping_round"},
        {"max_tree_output", "max_delta_step"}, {"max_leaf_output", "max_delta_step"}, {"reg_alpha", "lambda_l1"},
        {"reg_lambda", "lambda_l2"}, {"lambda", "lambda_l2"}, {"min_split_gain", "min_gain_to_split"},
        {"rate_drop", "drop_rate"}, {"topk", "top_k"}, {"verbose", "verbosity"},
        {"subsample_for_bin", "bin_construct_sample_cnt"}, {"data_seed", "data_random_seed"},
        {"is_pre_partition", "pre_partition"}, {"is_enable_bundle", "enable_bundle"}, {"bundle", "enable_bundle"}, {"cat_feature", "categorical_feature"},
        {"categorical_column", "categorical_feature"}, {"cat_column", "categorical_feature"},
        {"num_classes", "num_class"}, {"unbalance", "is_unbalance"}, {"unbalanced_sets", "is_unbalance"},
        {"max_position", "lambdarank_truncation_level"}, {"metrics", "metric"}, {"metric_types", "metric"},
        {"ndcg_eval_at", "eval_at"}, {"ndcg_at", "eval_at"}, {"map_eval_at", "eval_at"}, {"map_at", "eval_at"},
        {"fs", "forcedsplits_filename"}, {"forced_splits_filename", "forcedsplits_filename"},
        {"forced_splits_file", "forcedsplits_filename"}, {"forced_splits", "forcedsplits_filename"},
        {"num_machine", "num_machines"}, {"local_port", "local_listen_port"}, {"port", "local_listen_port"}};
    return a;
  }
  static std::string CanonObjective(const std::string& o) {
    if (o == "regression" || o == "regression_l2" || o == "l2" || o == "mean_squared_error" || o == "mse" ||
        o == "l2_root" || o == "root_mean_squared_error" || o == "rmse")
      return "regression";
    if (o == "softmax") return "multiclass";
    if (o == "multiclass_ova" || o == "ova" || o == "ovr") return "multiclassova";
    if (o == "xentropy") return "cross_entropy";
    if (o == "xentlambda") return "cross_entropy_lambda";
    if (o == "rank" ) return "lambdarank";
    if (o == "xendcg" || o == "xe_ndcg" || o == "xe_ndcg_mart" || o == "xendcg_mart") return "rank_xendcg";
    if (o == "l1" || o == "mean_absolute_error" || o == "mae") return "regression_l1";
    if (o == "mean_absolute_percentage_error") return "mape";
    return o;
  }
  static std::string CanonMetric(const std::string& m) {
    if (m == "regression" || m == "regression_l2" || m == "l2" || m == "mean_squared_error" || m == "mse") return "l2";
    if (m == "l2_root" || m == "root_mean_squared_error" || m == "rmse") return "rmse";
    if (m == "regression_l1" || m == "l1" || m == "mean_absolute_error" || m == "mae") return "l1";
    if (m == "binary_logloss" || m == "binary") return "binary_logloss";
    if (m == "multi_logloss" || m == "multiclass" || m == "softmax" || m == "multiclassova" || m == "multiclass_ova" ||
        m == "ova" || m == "ovr")
      return "multi_logloss";
    if (m == "ndcg" || m == "lambdarank" || m == "rank_xendcg" || m == "xendcg" || m == "xe_ndcg" || m == "xe_ndcg_mart" || m == "xendcg_mart")
      return "ndcg";
    if (m == "map" || m == "mean_average_precision") return "map";
    if (m == "xentropy" || m == "cross_entropy") return "cross_entropy";
    if (m == "xentlambda" || m == "cross_entropy_lambda") return "cross_entropy_lambda";
    if (m == "kldiv" || m == "kullback_leibler") return "kullback_leibler";
    if (m == "mean_absolute_percentage_error") return "mape";
    return m;
  }
  void Set(const std::map<std::string, std::string>& kv) {
    for (auto& p : kv) raw[p.first] = p.second;
    Refresh();
  }
  void Parse(const char* s) {
    if (!s) { Refresh(); return; }
    std::istringstream is(s);
    std::string tok;
    while (is >> tok) {
      size_t p = tok.find('=');
      if (p == std::string::npos) continue;
      std::string k = tok.substr(0, p), v = tok.substr(p + 1);
      auto it = Aliases().find(k);
      if (it != Aliases().end()) k = it->second;
      raw[k] = v;
    }
    Refresh();
  }
  // "[0,1,2],[2,3]" -> {{0,1,2},{2,3}} ([UPSTREAM] Common::StringToArrayofArrays); false unless the value is a comma-separated list of
  // bracketed, comma-separated integer lists with no empty item.  An empty value is the empty list; "[]" is an empty set.
  static bool ParseSets(const std::string& s, std::vector<std::vector<int>>* out) {
    out->clear();
    for (size_t i = 0; i < s.size();) {
      const size_t close = s.find(']', i);
      if (s[i] != '[' || close == std::string::npos) return false;
      std::vector<int> set;
      const std::string inner = s.substr(i + 1, close - i - 1);
      if (!inner.empty() && inner.back() == ',') return false;      // getline would drop the empty last item
      std::stringstream ss(inner);
      std::string x;
      while (std::getline(ss, x, ',')) {
        char* end = nullptr;
        const long long v = std::strtoll(x.c_str(), &end, 10);
        if (x.empty() || *end != '\0' || v < INT_MIN || v > INT_MAX) return false;
        set.push_back(static_cast<int>(v));
      }
      out->push_back(std::move(set));
      i = close + 1;
      if (i < s.size() && (s[i] != ',' || ++i == s.size())) return false;
    }
    return true;
  }
  template <typename T, typename F>
  static void SplitList(const std::string& s, std::vector<T>* out, F conv) {
    out->clear();
    std::stringstream ss(s);
    std::string x;
    while (std::getline(ss, x, ',')) if (!x.empty()) out->push_back(conv(x));
  }
  void Refresh() {
    auto I = [&](const char* k, int* d) { auto it = raw.find(k); if (it != raw.end() && !it->second.empty()) *d = std::atoi(it->second.c_str()); };
    auto D = [&](const char* k, double* d) { auto it = raw.find(k); if (it != raw.end() && !it->second.empty()) *d = std::atof(it->second.c_str()); };
    auto B = [&](const char* k, bool* d) { auto it = raw.find(k); if (it != raw.end() && !it->second.empty()) *d = ParseBool(it->second); };
    auto S = [&](const char* k, std::string* d) { auto it = raw.find(k); if (it != raw.end() && !it->second.empty()) *d = it->second; };
    S("objective", &objective); objective = CanonObjective(objective);
    S("boosting", &boosting); S("tree_learner", &tree_learner);
    if (boosting == "gbrt") boosting = "gbdt";
    if (boosting == "random_forest") boosting = "rf";
    if (tree_learner == "data" || tree_learner == "data_parallel") tree_learner = "data";
    else if (tree_learner == "voting" || tree_learner == "voting_parallel") tree_learner = "voting";
    else if (tree_learner == "feature" || tree_learner == "feature_parallel") tree_learner = "feature";
    I("num_iterations", &num_iterations); D("learning_rate", &learning_rate); I("num_leaves", &num_leaves);
    I("num_threads", &num_threads); I("max_depth", &max_depth); I("min_data_in_leaf", &min_data_in_leaf);
    D("min_sum_hessian_in_leaf", &min_sum_hessian_in_leaf); D("bagging_fraction", &bagging_fraction);
    D("pos_bagging_fraction", &pos_bagging_fraction); D("neg_bagging_fraction", &neg_bagging_fraction);
    I("bagging_freq", &bagging_freq); I("bagging_seed", &bagging_seed); D("feature_fraction", &feature_fraction);
    I("feature_fraction_seed", &feature_fraction_seed); D("feature_fraction_bynode", &feature_fraction_bynode);
    I("early_stopping_round", &early_stopping_round);
    B("extra_trees", &extra_trees); I("extra_seed", &extra_seed);
    S("monotone_constraints_method", &monotone_constraints_method); D("monotone_penalty", &monotone_penalty);
    D("path_smooth", &path_smooth);
    B("use_quantized_grad", &use_quantized_grad); I("num_grad_quant_bins", &num_grad_quant_bins);
    B("quant_train_renew_leaf", &quant_train_renew_leaf); B("stochastic_rounding", &stochastic_rounding);
    D("refit_decay_rate", &refit_decay_rate);
    {   // an empty value clears it
      auto it = raw.find("forcedsplits_filename");
      forcedsplits_filename = it != raw.end() ? it->second : "";
    }
    D("max_delta_step", &max_delta_step); D("lambda_l1", &lambda_l1); D("lambda_l2", &lambda_l2);
    D("min_gain_to_split", &min_gain_to_split); D("cat_l2", &cat_l2); D("cat_smooth", &cat_smooth);
    I("max_cat_threshold", &max_cat_threshold); I("max_cat_to_onehot", &max_cat_to_onehot); I("min_data_per_group", &min_data_per_group);
    D("drop_rate", &drop_rate); I("max_drop", &max_drop); I("drop_seed", &drop_seed);
    D("skip_drop", &skip_drop); B("xgboost_dart_mode", &xgboost_dart_mode); B("uniform_drop", &uniform_drop);
    D("top_rate", &top_rate); D("other_rate", &other_rate); I("top_k", &top_k); I("verbosity", &verbosity);
    I("max_bin", &max_bin); I("min_data_in_bin", &min_data_in_bin); I("bin_construct_sample_cnt", &bin_construct_sample_cnt);
    I("data_random_seed", &data_random_seed); B("use_missing", &use_missing); B("zero_as_missing", &zero_as_missing);
    B("feature_pre_filter", &feature_pre_filter); B("pre_partition", &pre_partition); B("enable_bundle", &enable_bundle);
    S("max_bin_by_feature", &max_bin_by_feature);
    I("num_class", &num_class); B("is_unbalance", &is_unbalance); D("scale_pos_weight", &scale_pos_weight);
    D("sigmoid", &sigmoid); B("boost_from_average", &boost_from_average); D("alpha", &alpha);
    D("tweedie_variance_power", &tweedie_variance_power); D("fair_c", &fair_c); D("poisson_max_delta_step", &poisson_max_delta_step); I("objective_seed", &objective_seed);
    I("lambdarank_truncation_level", &lambdarank_truncation_level);
    B("lambdarank_norm", &lambdarank_norm); I("num_machines", &num_machines);
    D("lambdarank_position_bias_regularization", &lambdarank_position_bias_regularization);
    B("pred_early_stop", &pred_early_stop); I("pred_early_stop_freq", &pred_early_stop_freq); D("pred_early_stop_margin", &pred_early_stop_margin);
    {
      auto it = raw.find("label_gain");
      if (it != raw.end() && !it->second.empty()) SplitList(it->second, &label_gain, [](const std::string& x) { return std::atof(x.c_str()); });
      it = raw.find("eval_at");
      if (it != raw.end() && !it->second.empty()) SplitList(it->second, &eval_at, [](const std::string& x) { return std::atoi(x.c_str()); });
      it = raw.find("auc_mu_weights");
      if (it != raw.end() && !it->second.empty()) SplitList(it->second, &auc_mu_weights, [](const std::string& x) { return std::atof(x.c_str()); });
      it = raw.find("monotone_constraints");      // an empty value clears the list
      if (it != raw.end()) SplitList(it->second, &monotone_constraints, [](const std::string& x) { return std::atoi(x.c_str()); });
      it = raw.find("interaction_constraints");   // an empty value clears the list
      if (it != raw.end()) {
        interaction_constraints_malformed.clear();
        if (!ParseSets(it->second, &interaction_constraints)) { interaction_constraints.clear(); interaction_constraints_malformed = it->second; }
      }
      it = raw.find("categorical_feature");
      if (it != raw.end() && !it->second.empty()) SplitList(it->second, &categorical_feature, [](const std::string& x) { return std::atoi(x.c_str()); });
    }
    if (eval_at.empty()) eval_at = {1, 2, 3, 4, 5};
    // [UPSTREAM] Config::CheckParamConflict: a smoothed leaf needs at least two rows.  min_data_in_leaf is re-read from raw above, so a
    // reset that turns smoothing off gives back the value the caller set.
    if (path_smooth > kPathSmoothEps && min_data_in_leaf < 2) min_data_in_leaf = 2;
    // metric resolution: empty => the objective's default metric (SURVEY.md B.5)
    metric.clear();
    auto it = raw.find("metric");
    metric_given = it != raw.end() && !it->second.empty();
    std::vector<std::string> names;
    if (metric_given) SplitList(it->second, &names, [](const std::string& x) { return x; });
    else names.push_back(objective);
    for (auto& m : names) {
      std::string c = CanonMetric(m);
      if (c == "None" || c == "none" || c == "null" || c == "na" || c == "custom") continue;
      bool dup = false;
      for (auto& e : metric) dup |= (e == c);
      if (!dup) metric.push_back(c);
    }
  }
  static std::string Num(double v) {
    std::ostringstream s;
    s << v;
    return s.str();
  }
  // [UPSTREAM Config::SaveMembersToString order]; the reference's tests grep this block, e.g.
  // "[lambda_l1: 0.1]" (VerifyLightGBMClassifier.scala:273-275) and "learning_rate: 0.005" (:509).
  std::string ToString() const {
    std::ostringstream s;
    auto join_i = [](const std::vector<int>& v) { std::string r; for (size_t i = 0; i < v.size(); ++i) r += (i ? "," : "") + std::to_string(v[i]); return r; };
    auto join_d = [](const std::vector<double>& v) { std::string r; for (size_t i = 0; i < v.size(); ++i) r += (i ? "," : "") + Num(v[i]); return r; };
    auto join_sets = [&](const std::vector<std::vector<int>>& v) { std::string r; for (size_t i = 0; i < v.size(); ++i) r += (i ? ",[" : "[") + join_i(v[i]) + "]"; return r; };
    auto join_s = [](const std::vector<std::string>& v) { std::string r; for (size_t i = 0; i < v.size(); ++i) r += (i ? "," : "") + v[i]; return r; };
    std::string tl = tree_learner == "data" ? "data" : tree_learner;
    s << "[boosting: " << boosting << "]\n[objective: " << objective << "]\n[metric: " << join_s(metric) << "]\n";
    s << "[tree_learner: " << tl << "]\n[device_type: cuda_b200]\n[data: ]\n[valid: ]\n";
    s << "[num_iterations: " << num_iterations << "]\n[learning_rate: " << Num(learning_rate) << "]\n";
    s << "[num_leaves: " << num_leaves << "]\n[num_threads: " << num_threads << "]\n[deterministic: 1]\n";
    s << "[force_col_wise: 0]\n[force_row_wise: 0]\n[histogram_pool_size: -1]\n[max_depth: " << max_depth << "]\n";
    s << "[min_data_in_leaf: " << min_data_in_leaf << "]\n[min_sum_hessian_in_leaf: " << Num(min_sum_hessian_in_leaf) << "]\n";
    s << "[bagging_fraction: " << Num(bagging_fraction) << "]\n[pos_bagging_fraction: " << Num(pos_bagging_fraction) << "]\n";
    s << "[neg_bagging_fraction: " << Num(neg_bagging_fraction) << "]\n[bagging_freq: " << bagging_freq << "]\n";
    s << "[bagging_seed: " << bagging_seed << "]\n[feature_fraction: " << Num(feature_fraction) << "]\n";
    s << "[feature_fraction_bynode: " << Num(feature_fraction_bynode) << "]\n[feature_fraction_seed: " << feature_fraction_seed << "]\n[extra_trees: " << extra_trees << "]\n[extra_seed: " << extra_seed << "]\n";
    s << "[early_stopping_round: " << early_stopping_round << "]\n[first_metric_only: 0]\n";
    s << "[max_delta_step: " << Num(max_delta_step) << "]\n[lambda_l1: " << Num(lambda_l1) << "]\n[lambda_l2: " << Num(lambda_l2) << "]\n";
    s << "[linear_lambda: 0]\n[min_gain_to_split: " << Num(min_gain_to_split) << "]\n[drop_rate: " << Num(drop_rate) << "]\n";
    s << "[max_drop: " << max_drop << "]\n[skip_drop: " << Num(skip_drop) << "]\n[xgboost_dart_mode: " << xgboost_dart_mode << "]\n";
    s << "[uniform_drop: " << uniform_drop << "]\n[drop_seed: " << drop_seed << "]\n[top_rate: " << Num(top_rate) << "]\n[other_rate: " << Num(other_rate) << "]\n";
    s << "[min_data_per_group: " << min_data_per_group << "]\n[max_cat_threshold: " << max_cat_threshold << "]\n[cat_l2: " << Num(cat_l2) << "]\n";
    s << "[cat_smooth: " << Num(cat_smooth) << "]\n[max_cat_to_onehot: " << max_cat_to_onehot << "]\n";
    s << "[top_k: " << top_k << "]\n[monotone_constraints: " << join_i(monotone_constraints) << "]\n";
    s << "[monotone_constraints_method: " << monotone_constraints_method << "]\n[monotone_penalty: " << Num(monotone_penalty) << "]\n";
    s << "[feature_contri: ]\n[forcedsplits_filename: " << forcedsplits_filename << "]\n[refit_decay_rate: " << Num(refit_decay_rate) << "]\n[cegb_tradeoff: 1]\n[cegb_penalty_split: 0]\n";
    s << "[cegb_penalty_feature_lazy: ]\n[cegb_penalty_feature_coupled: ]\n[path_smooth: " << Num(path_smooth) << "]\n";
    s << "[interaction_constraints: " << join_sets(interaction_constraints) << "]\n";
    if (use_quantized_grad)      // only when on, so every other model text stays as it was
      s << "[use_quantized_grad: 1]\n[num_grad_quant_bins: " << num_grad_quant_bins << "]\n[quant_train_renew_leaf: " << quant_train_renew_leaf
        << "]\n[stochastic_rounding: " << stochastic_rounding << "]\n";
    s << "[verbosity: " << verbosity << "]\n[saved_feature_importance_type: 0]\n[linear_tree: 0]\n[max_bin: " << max_bin << "]\n";
    s << "[max_bin_by_feature: " << max_bin_by_feature << "]\n[min_data_in_bin: " << min_data_in_bin << "]\n";
    s << "[bin_construct_sample_cnt: " << bin_construct_sample_cnt << "]\n[data_random_seed: " << data_random_seed << "]\n";
    s << "[is_enable_sparse: 1]\n[enable_bundle: " << enable_bundle << "]\n[use_missing: " << use_missing << "]\n[zero_as_missing: " << zero_as_missing << "]\n";
    s << "[feature_pre_filter: " << feature_pre_filter << "]\n[pre_partition: " << pre_partition << "]\n[two_round: 0]\n[header: 0]\n";
    s << "[label_column: ]\n[weight_column: ]\n[group_column: ]\n[ignore_column: ]\n[categorical_feature: " << join_i(categorical_feature) << "]\n";
    s << "[forcedbins_filename: ]\n[objective_seed: " << objective_seed << "]\n[num_class: " << num_class << "]\n[is_unbalance: " << is_unbalance << "]\n";
    s << "[scale_pos_weight: " << Num(scale_pos_weight) << "]\n[sigmoid: " << Num(sigmoid) << "]\n[boost_from_average: " << boost_from_average << "]\n";
    s << "[reg_sqrt: 0]\n[alpha: " << Num(alpha) << "]\n[fair_c: " << Num(fair_c) << "]\n[poisson_max_delta_step: " << Num(poisson_max_delta_step) << "]\n";
    s << "[tweedie_variance_power: " << Num(tweedie_variance_power) << "]\n[lambdarank_truncation_level: " << lambdarank_truncation_level << "]\n";
    s << "[lambdarank_norm: " << lambdarank_norm << "]\n[label_gain: " << join_d(label_gain) << "]\n";
    if (lambdarank_position_bias_regularization != 0.0)      // only when set, so every other model text stays as it was
      s << "[lambdarank_position_bias_regularization: " << Num(lambdarank_position_bias_regularization) << "]\n";
    s << "[eval_at: " << join_i(eval_at) << "]\n";
    s << "[multi_error_top_k: 1]\n[auc_mu_weights: " << join_d(auc_mu_weights) << "]\n[num_machines: " << num_machines << "]\n[local_listen_port: 12400]\n";
    s << "[time_out: 120]\n[machine_list_filename: ]\n[machines: ]\n[gpu_platform_id: -1]\n[gpu_device_id: -1]\n[gpu_use_dp: 0]\n[num_gpu: 1]";
    return s.str();
  }
};

}  // namespace b200gbm
