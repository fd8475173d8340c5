// Training objective of a Booster, chosen once from the config.  Everything that depends on it lives here: the config and label checks,
// class counts and weights, the tables of the k_grad_* kernels (kernels.cuh), the init score, the model header and the leaf-renewal parameters.
#pragma once
#include <algorithm>
#include <functional>
#include <numeric>
#include "engine.h"
#include "refit_kernels.cuh"      // k_refit_leaf_sums: the per-position sums of the position factors' update

namespace b200gbm {

enum class ObjectiveKind { kRegression, kHuber, kFair, kPoisson, kGamma, kTweedie, kRegressionL1, kQuantile, kMape, kBinary, kMulticlass,
                           kMulticlassOva, kCrossEntropy, kCrossEntropyLambda, kLambdarank, kRankXendcg };

// Each objective the engine trains: its canonical name (Config has resolved the aliases) and the `kind` argument it passes to
// k_grad_regvar (huber 1 .. tweedie 5) or k_grad_percentile (regression_l1 1, quantile 2, mape 3); 0 for the other kernels
struct ObjectiveName { const char* name; ObjectiveKind kind; int grad_kind; };
constexpr ObjectiveName kObjectiveNames[] = {
    {"regression", ObjectiveKind::kRegression, 0}, {"huber", ObjectiveKind::kHuber, 1}, {"fair", ObjectiveKind::kFair, 2},
    {"poisson", ObjectiveKind::kPoisson, 3}, {"gamma", ObjectiveKind::kGamma, 4}, {"tweedie", ObjectiveKind::kTweedie, 5},
    {"regression_l1", ObjectiveKind::kRegressionL1, 1}, {"quantile", ObjectiveKind::kQuantile, 2}, {"mape", ObjectiveKind::kMape, 3},
    {"binary", ObjectiveKind::kBinary, 0}, {"multiclass", ObjectiveKind::kMulticlass, 0}, {"multiclassova", ObjectiveKind::kMulticlassOva, 0},
    {"cross_entropy", ObjectiveKind::kCrossEntropy, 0}, {"cross_entropy_lambda", ObjectiveKind::kCrossEntropyLambda, 0},
    {"lambdarank", ObjectiveKind::kLambdarank, 0}, {"rank_xendcg", ObjectiveKind::kRankXendcg, 0}};
inline ObjectiveKind ParseObjectiveKind(const std::string& name) {
  for (const ObjectiveName& o : kObjectiveNames) if (name == o.name) return o.kind;
  Fatal("Unknown/unsupported objective type name: " + name);
}
inline int GradKernelKind(ObjectiveKind kind) {
  for (const ObjectiveName& o : kObjectiveNames) if (kind == o.kind) return o.grad_kind;
  return 0;
}

// [UPSTREAM DCGCalculator] label gains (default 2^i - 1) and position discounts 1 / log2(2 + i) for positions [0, max_q], host log2
inline std::vector<double> LabelGain(const Config& cfg) {
  std::vector<double> lg = cfg.label_gain;
  if (lg.empty()) { lg.push_back(0.0); for (int i = 1; i < 31; ++i) lg.push_back(static_cast<double>((1 << i) - 1)); }
  return lg;
}
inline std::vector<double> DcgDiscount(int max_q) {
  std::vector<double> disc(static_cast<size_t>(std::max(max_q, 1)) + 1);
  for (size_t i = 0; i < disc.size(); ++i) disc[i] = 1.0 / std::log2(2.0 + i);
  return disc;
}

// dynamic shared memory of k_grad_lambdarank: per-document arrays + the pair matrix of one j-tile
inline size_t LambdarankSmem(int max_q, int truncation) {
  return static_cast<size_t>(max_q) * (8 + 8 + 4 + 4 + 4 + 4) + 8 + static_cast<size_t>(truncation) * (lr_tile(truncation) + 1) * 8;
}

// Init score of regression_l1 / quantile / mape [LightGBM regression_objective.hpp PercentileFun / WeightedPercentileFun, T = label_t]:
// the alpha percentile counted from the top of the descending order d[]: fp = (cnt-1)(1-alpha), interpolation between d[int(fp)] and
// d[int(fp)+1]; weighted: upper_bound on the running weight sum.
inline float LabelPercentile(const float* y, int cnt, double alpha) {
  if (cnt <= 1) return y[0];
  const double float_pos = static_cast<double>(cnt - 1) * (1.0 - alpha);
  const int pos = static_cast<int>(float_pos) + 1;
  if (pos < 1) return *std::max_element(y, y + cnt);
  if (pos >= cnt) return *std::min_element(y, y + cnt);
  std::vector<float> v(y, y + cnt);
  std::nth_element(v.begin(), v.begin() + pos, v.end(), std::greater<float>());      // v[pos] = (pos+1)-th largest, larger ones before it
  const float v2 = v[pos], v1 = *std::min_element(v.begin(), v.begin() + pos);
  return static_cast<float>(v1 - (v1 - v2) * (float_pos - (pos - 1)));
}
inline float LabelWeightedPercentile(const float* y, const float* w, int cnt, double alpha) {
  if (cnt <= 1) return y[0];
  std::vector<int> order(cnt);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return y[a] < y[b]; });
  std::vector<double> cdf(cnt);
  cdf[0] = w[order[0]];
  for (int i = 1; i < cnt; ++i) cdf[i] = cdf[i - 1] + w[order[i]];
  const double threshold = cdf[cnt - 1] * alpha;
  size_t pos = std::upper_bound(cdf.begin(), cdf.end(), threshold) - cdf.begin();
  pos = std::min(pos, static_cast<size_t>(cnt - 1));
  if (pos == 0 || pos == static_cast<size_t>(cnt - 1)) return y[order[pos]];
  const float v1 = y[order[pos - 1]], v2 = y[order[pos]];
  if (cdf[pos + 1] - cdf[pos] >= 1.0f) return static_cast<float>((threshold - cdf[pos]) / (cdf[pos + 1] - cdf[pos]) * (v2 - v1) + v1);
  return v2;
}

class Objective {
  using Kind = ObjectiveKind;

 public:
  // Checks the name, quantile's alpha, the class count of multiclass / multiclassova and the query information of the ranking objectives.  `cfg` is
  // read again by every later call, so that a parameter reset reaches the gradients as it reaches the rest of the booster.
  Objective(const Config& cfg, const Dataset& train) : cfg_(cfg), train_(train), kind_(ParseObjectiveKind(cfg.objective)) {
    const bool multi = kind_ == Kind::kMulticlass || kind_ == Kind::kMulticlassOva;
    if (kind_ == Kind::kQuantile && !(cfg.alpha > 0.0 && cfg.alpha < 1.0)) Fatal("Check failed: alpha_ > 0 && alpha_ < 1");
    if (multi && cfg.num_class < 2) Fatal("Number of classes should be specified and greater than 1 for multiclass training");
    if ((kind_ == Kind::kLambdarank || kind_ == Kind::kRankXendcg) && train.query_boundaries.empty()) Fatal("Ranking tasks require query information");
    K_ = multi ? cfg.num_class : 1;
    if (kind_ == Kind::kQuantile) renew_alpha_ = static_cast<double>(static_cast<float>(cfg.alpha));     // quantile keeps alpha as score_t
  }
  ObjectiveKind kind() const { return kind_; }
  int NumTreePerIteration() const { return K_; }
  // every row's hessian is 1: unweighted regression / regression_l1 / quantile / mape (GOSS makes it vary again)
  bool ConstHessian() const { return (kind_ == Kind::kRegression || RenewsLeaves()) && train_.weight.empty(); }
  bool NeedTrain(int k) const { return need_train_[k] != 0; }      // false: class k gets a constant tree (one-sided labels, or a prior of 0 or 1)
  // regression_l1 / quantile / mape renew each leaf output to the (weighted) alpha percentile of its residuals
  bool RenewsLeaves() const { return kind_ == Kind::kRegressionL1 || kind_ == Kind::kQuantile || kind_ == Kind::kMape; }
  double RenewAlpha() const { return renew_alpha_; }
  const float* RenewWeights() const { return kind_ == Kind::kMape ? label_weight_.p : (train_.weight.empty() ? nullptr : train_.d_weight.p); }

  // label and weight checks, the global class counts (all-reduced in the same order on every rank) and the device tables
  void Init(cudaStream_t s) {
    stream_ = s; const int n = train_.num_data;
    const std::vector<float>& y = train_.label, &w = train_.weight;
    need_train_.assign(K_, 1);
    auto label_class = [&](float v) {      // multiclass / multiclassova
      const int l = static_cast<int>(v);
      if (l < 0 || l >= K_) Fatal("Label must be in [0, " + std::to_string(K_) + "), but found " + std::to_string(l) + " in label");
      return l;
    };
    if (kind_ == Kind::kPoisson || kind_ == Kind::kGamma || kind_ == Kind::kTweedie) {
      for (int i = 0; i < n; ++i) if (y[i] < 0) Fatal("[" + cfg_.objective + "]: at least one target label is negative");
    } else if (kind_ == Kind::kMape) {       // [LightGBM RegressionMAPELOSS::Init] label_weight = 1 / max(1, |label|) (* weight)
      label_weight_host_.resize(n);
      for (int i = 0; i < n; ++i) label_weight_host_[i] = 1.0f / std::max(1.0f, std::fabs(y[i])) * (w.empty() ? 1.0f : w[i]);
      label_weight_.Alloc(n); label_weight_.Upload(label_weight_host_.data(), n, s);
    } else if (kind_ == Kind::kBinary) {
      double cnt[2] = {0, 0}; for (int i = 0; i < n; ++i) cnt[y[i] > 0 ? 1 : 0] += 1;
      AllReduceHost(cnt, 2, ncclSum, s);          // global class counts (R14)
      need_train_[0] = !(cnt[0] == 0 || cnt[1] == 0);
      ClassWeights(cnt[1], cnt[0], binary_w_);
    } else if (kind_ == Kind::kMulticlass) {
      class_init_probs_.assign(K_ + 1, 0.0);
      for (int i = 0; i < n; ++i) { const double wi = w.empty() ? 1.0 : w[i]; class_init_probs_[label_class(y[i])] += wi; class_init_probs_[K_] += wi; }
      AllReduceHost(class_init_probs_.data(), K_ + 1, ncclSum, s);
      for (int k = 0; k < K_; ++k) { class_init_probs_[k] /= class_init_probs_[K_]; need_train_[k] = !(std::fabs(class_init_probs_[k]) <= kEps || std::fabs(class_init_probs_[k]) >= 1.0 - kEps); }
    } else if (kind_ == Kind::kMulticlassOva) {       // [UPSTREAM MulticlassOVA::Init]: one BinaryLogloss::Init per class on (label == k)
      std::vector<double> cnt(K_, 0.0), cw(2 * static_cast<size_t>(K_), 1.0);
      for (int i = 0; i < n; ++i) cnt[label_class(y[i])] += 1;
      double total = n;
      AllReduceHost(cnt.data(), K_, ncclSum, s);
      AllReduceHost(&total, 1, ncclSum, s);
      for (int k = 0; k < K_; ++k) { need_train_[k] = !(cnt[k] == 0 || total - cnt[k] == 0); ClassWeights(cnt[k], total - cnt[k], &cw[2 * k]); }
      ova_w_.Alloc(cw.size()); ova_w_.Upload(cw.data(), cw.size(), s);
      ova_need_.Alloc(K_); ova_need_.Upload(need_train_.data(), K_, s);
      B200_CUDA(cudaStreamSynchronize(s));
    } else if (kind_ == Kind::kCrossEntropy) {      // [UPSTREAM CrossEntropy::Init]
      for (int i = 0; i < n; ++i) if (!(y[i] >= 0.0f && y[i] <= 1.0f)) Fatal("[cross_entropy]: does not tolerate label " + std::to_string(y[i]) + " outside [0, 1]");
      if (!w.empty()) {
        double sw = 0; for (int i = 0; i < n; ++i) { if (w[i] < 0) Fatal("[cross_entropy]: at least one weight is negative"); sw += w[i]; }
        if (!(sw > 0)) Fatal("[cross_entropy]: sum of weights is zero");
      }
    } else if (kind_ == Kind::kCrossEntropyLambda) {      // [UPSTREAM CrossEntropyLambda::Init]
      for (int i = 0; i < n; ++i) if (!(y[i] >= 0.0f && y[i] <= 1.0f)) Fatal("[cross_entropy_lambda]: does not tolerate label " + std::to_string(y[i]) + " outside [0, 1]");
      for (int i = 0; i < static_cast<int>(w.size()); ++i) if (!(w[i] > 0.0f)) Fatal("[cross_entropy_lambda]: at least one weight is non-positive");
    } else if (kind_ == Kind::kRankXendcg) {
      // one LCG per (rank-local) query, seeded objective_seed + q [UPSTREAM RankXENDCG::Init], and the jump table of its first max_q draws
      const int nq = static_cast<int>(train_.query_boundaries.size()) - 1;
      std::vector<unsigned> st(nq);
      int max_q = 1;
      for (int q = 0; q < nq; ++q) {
        st[q] = static_cast<unsigned>(cfg_.objective_seed + q);
        max_q = std::max(max_q, train_.query_boundaries[q + 1] - train_.query_boundaries[q]);
      }
      std::vector<unsigned> jump(2 * static_cast<size_t>(max_q));      // [mul][max_q], [add][max_q]: x_{j+1} = mul[j] x_0 + add[j]
      unsigned a = 1, c = 0;
      for (int j = 0; j < max_q; ++j) { a = a * 214013u; c = c * 214013u + 2531011u; jump[j] = a; jump[max_q + j] = c; }
      xe_max_q_ = max_q;
      xe_state_.Alloc(nq); xe_state_.Upload(st.data(), nq, s);
      xe_jump_.Alloc(jump.size()); xe_jump_.Upload(jump.data(), jump.size(), s);
      xe_scratch_.Alloc(2 * static_cast<size_t>(n));
      B200_CUDA(cudaStreamSynchronize(s));
    } else if (kind_ == Kind::kLambdarank) {
      const std::vector<double> lg = LabelGain(cfg_);
      const int nq = static_cast<int>(train_.query_boundaries.size()) - 1;
      std::vector<double> imd(nq);
      for (int q = 0; q < nq; ++q) {
        const int b = train_.query_boundaries[q], cnt = train_.query_boundaries[q + 1] - b;
        lr_max_q_ = std::max(lr_max_q_, cnt);
        std::vector<int> label_cnt(lg.size(), 0);
        for (int i = 0; i < cnt; ++i) {
          int l = static_cast<int>(train_.label[b + i]);
          if (l < 0 || l >= static_cast<int>(lg.size())) Fatal("Label excel the max range " + std::to_string(lg.size()) + " for lambdarank");
          ++label_cnt[l];
        }
        int top = static_cast<int>(lg.size()) - 1, k = std::min(cfg_.lambdarank_truncation_level, cnt);
        double m = 0;
        for (int j = 0; j < k; ++j) {
          while (top > 0 && label_cnt[top] <= 0) --top;
          m += (1.0 / std::log2(2.0 + j)) * lg[top];      // discount_[j] * label_gain_[top] as [UPSTREAM DCGCalculator::CalMaxDCGAtK]
          --label_cnt[top];
        }
        imd[q] = m > 0.0 ? 1.0 / m : m;
      }
      lr_inv_max_dcg_.Alloc(nq); lr_inv_max_dcg_.Upload(imd.data(), nq, s);
      lr_label_gain_.Alloc(lg.size()); lr_label_gain_.Upload(lg.data(), lg.size(), s);
      const size_t bins_n = 1024 * 1024;
      lr_min_in_ = -50.0 / cfg_.sigmoid / 2; lr_max_in_ = 50.0 / cfg_.sigmoid / 2; lr_idx_factor_ = bins_n / (lr_max_in_ - lr_min_in_);
      std::vector<float> tab(bins_n);
      for (size_t i = 0; i < bins_n; ++i) tab[i] = static_cast<float>(1.0 / (1.0 + std::exp((i / lr_idx_factor_ + lr_min_in_) * cfg_.sigmoid)));
      lr_sig_table_.Alloc(bins_n); lr_sig_table_.Upload(tab.data(), bins_n, s);
      const std::vector<double> disc = DcgDiscount(lr_max_q_);
      lr_discount_.Alloc(disc.size()); lr_discount_.Upload(disc.data(), disc.size(), s);
      B200_CUDA(cudaStreamSynchronize(s));
      if (cfg_.lambdarank_truncation_level < 1 || cfg_.lambdarank_truncation_level > 180) Fatal("lambdarank_truncation_level should be in [1, 180]");
      size_t smem = LambdarankSmem(lr_max_q_, cfg_.lambdarank_truncation_level);
      if (smem > 200 * 1024) Fatal("a query group is too large for the lambdarank kernel");
      B200_CUDA(cudaFuncSetAttribute(k_grad_lambdarank, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(std::max<size_t>(smem, 1024))));
    }
    if (kind_ == Kind::kLambdarank || kind_ == Kind::kRankXendcg) InitPositions();
  }

  // init score of class k, the same on every rank
  double BoostFromScore(int k) {
    if (kind_ == Kind::kMulticlass) return std::log(std::max(kEps, class_init_probs_[k]));
    if (kind_ == Kind::kLambdarank || kind_ == Kind::kRankXendcg) return 0.0;
    const int n = train_.num_data; double v;
    const float* y = train_.label.data(); const std::vector<float>& w = train_.weight;
    if (kind_ == Kind::kMape) v = LabelWeightedPercentile(y, label_weight_host_.data(), n, 0.5);
    else if (RenewsLeaves()) v = w.empty() ? LabelPercentile(y, n, renew_alpha_) : LabelWeightedPercentile(y, w.data(), n, renew_alpha_);
    else {      // weighted means of the label (binary: of label > 0, multiclassova: of label == k)
      double s[2] = {0, 0};
      for (int i = 0; i < n; ++i) {
        const double wi = w.empty() ? 1.0 : static_cast<double>(w[i]);
        s[0] += wi * (kind_ == Kind::kBinary ? (y[i] > 0) : kind_ == Kind::kMulticlassOva ? (static_cast<int>(y[i]) == k) : y[i]); s[1] += wi;
      }
      if (kind_ == Kind::kBinary || kind_ == Kind::kMulticlassOva || kind_ == Kind::kCrossEntropy) {      // [UPSTREAM BinaryLogloss / CrossEntropy::BoostFromScore]
        AllReduceHost(s, 2, ncclSum, stream_);
        const double pavg = std::max(std::min(s[0] / s[1], 1.0 - kEps), kEps);
        return std::log(pavg / (1.0 - pavg)) / (kind_ == Kind::kCrossEntropy ? 1.0 : cfg_.sigmoid);
      }
      if (kind_ == Kind::kCrossEntropyLambda) {      // [UPSTREAM CrossEntropyLambda::BoostFromScore], global sums as cross_entropy
        AllReduceHost(s, 2, ncclSum, stream_);
        return std::log(std::expm1(s[0] / s[1]));
      }
      v = s[0] / s[1];
      if (kind_ == Kind::kPoisson || kind_ == Kind::kGamma || kind_ == Kind::kTweedie) v = v > 0 ? std::log(v) : -std::numeric_limits<double>::infinity();
    }
    if (Net().active && Net().world > 1) { AllReduceHost(&v, 1, ncclSum, stream_); v /= Net().world; }   // GlobalSyncUpByMean (R11)
    return v;
  }

  // advance: a training iteration, which moves rank_xendcg's random states on; false reads the gradients without changing them
  void LaunchGradients(const double* score, float* g, float* h, int num_sms, bool advance) const {
    const int n = train_.num_data, grid = num_sms * 8;
    const float *y = train_.d_label.p, *w = train_.weight.empty() ? nullptr : train_.d_weight.p;
    switch (kind_) {
      case Kind::kRegression: k_grad_l2<<<grid, 256, 0, stream_>>>(score, y, w, g, h, n); break;
      case Kind::kHuber: case Kind::kFair: case Kind::kPoisson: case Kind::kGamma: case Kind::kTweedie:
        k_grad_regvar<<<grid, 256, 0, stream_>>>(score, y, w, g, h, n, GradKernelKind(kind_), cfg_.alpha, cfg_.fair_c, cfg_.poisson_max_delta_step, cfg_.tweedie_variance_power); break;
      case Kind::kRegressionL1: case Kind::kQuantile: case Kind::kMape:
        k_grad_percentile<<<grid, 256, 0, stream_>>>(score, y, w, kind_ == Kind::kMape ? label_weight_.p : nullptr, g, h, n, GradKernelKind(kind_), static_cast<float>(cfg_.alpha)); break;
      case Kind::kBinary: if (need_train_[0]) k_grad_binary<<<grid, 256, 0, stream_>>>(score, y, w, g, h, n, cfg_.sigmoid, binary_w_[0], binary_w_[1]); break;
      case Kind::kMulticlass: k_grad_softmax<<<grid, 256, 0, stream_>>>(score, y, w, g, h, n, K_, static_cast<double>(K_) / (K_ - 1.0)); break;
      case Kind::kMulticlassOva: k_grad_ova<<<grid, 256, 0, stream_>>>(score, y, w, g, h, n, K_, cfg_.sigmoid, ova_w_.p, ova_need_.p); break;
      case Kind::kCrossEntropy: k_grad_xent<<<grid, 256, 0, stream_>>>(score, y, w, g, h, n); break;
      case Kind::kCrossEntropyLambda: k_grad_xentlambda<<<grid, 256, 0, stream_>>>(score, y, w, g, h, n); break;
      case Kind::kRankXendcg: {
        const int nq = static_cast<int>(train_.query_boundaries.size()) - 1;
        k_grad_xendcg<<<std::max(1, std::min(nq, num_sms * 16)), kXeThreads, 0, stream_>>>(score, PositionIds(), pos_bias_.p, y, w, train_.d_qb.p, nq,
                                                                                         xe_state_.p, xe_jump_.p, xe_jump_.p + xe_max_q_,
                                                                                         advance ? 1 : 0, xe_scratch_.p, n, g, h);
        break;
      }
      case Kind::kLambdarank: {
        const int nq = static_cast<int>(train_.query_boundaries.size()) - 1;
        const size_t smem = std::max<size_t>(LambdarankSmem(lr_max_q_, cfg_.lambdarank_truncation_level), 1024);
        k_grad_lambdarank<<<std::min(nq, num_sms * 16), kLrThreads, smem, stream_>>>(
            score, PositionIds(), pos_bias_.p, y, w, train_.d_qb.p, nq, lr_inv_max_dcg_.p, lr_label_gain_.p, lr_discount_.p, lr_sig_table_.p, 1024 * 1024, lr_min_in_,
            lr_max_in_, lr_idx_factor_, cfg_.sigmoid, cfg_.lambdarank_truncation_level, cfg_.lambdarank_norm ? 1 : 0, g, h, lr_max_q_); break;
      }
    }
    if (advance && !pos_values_.empty()) UpdatePositionBias(g, h, num_sms);
  }

  // the distinct position values (sorted, over every rank) and their factors; empty without a position field or for another objective
  void PositionBias(std::vector<int32_t>* values, std::vector<double>* factors) const {
    *values = pos_values_;
    factors->assign(pos_values_.size(), 0.0);
    if (pos_values_.empty()) return;
    pos_bias_.Download(factors->data(), factors->size(), stream_);
    B200_CUDA(cudaStreamSynchronize(stream_));
  }

  std::string ToString() const {      // objective= value of the model header
    if (kind_ == Kind::kBinary) return "binary sigmoid:" + Config::Num(cfg_.sigmoid);
    if (kind_ == Kind::kMulticlass) return "multiclass num_class:" + std::to_string(K_);
    if (kind_ == Kind::kMulticlassOva) return "multiclassova num_class:" + std::to_string(K_) + " sigmoid:" + Config::Num(cfg_.sigmoid);
    return cfg_.objective;
  }

 private:
  // [UPSTREAM BinaryLogloss::Init] {w_neg, w_pos}: is_unbalance weighs the smaller side up to the larger one, scale_pos_weight the positives
  void ClassWeights(double pos, double neg, double* cw) const {
    if (cfg_.is_unbalance && pos > 0 && neg > 0) { if (pos > neg) cw[0] = pos / neg; else cw[1] = neg / pos; }
    cw[1] *= cfg_.scale_pos_weight;
  }

  const int* PositionIds() const { return pos_values_.empty() ? nullptr : pos_id_.p; }

  // [UPSTREAM 4.1 Metadata::SetPosition, from knowledge] one factor per distinct position value, starting at 0.  The ids are global: the
  // sorted union of every rank's values, gathered padded to the largest count, so that every rank updates the same factors.  Every rank
  // of a ranking booster takes part in the first collective, so ranks that disagree on having the field all fail here.
  void InitPositions() {
    const int n = train_.num_data;
    std::vector<int32_t> local(train_.position);
    std::sort(local.begin(), local.end());
    local.erase(std::unique(local.begin(), local.end()), local.end());
    const bool has = !train_.position.empty();
    const bool net = Net().active && Net().world > 1;
    if (net) {
      double v[3] = {has ? 1.0 : 0.0, has ? -1.0 : 0.0, static_cast<double>(local.size())};      // max: any rank has it, not every rank has it
      AllReduceHost(v, 3, ncclMax, stream_);
      if (v[0] != -v[1]) Fatal("the position field is set on some ranks' training data and not on others; set it on every rank or on none");
      if (!has) return;
      const size_t stride = 1 + static_cast<size_t>(v[2]);      // [count, values padded with 0]
      std::vector<int32_t> send(stride, 0), recv(stride * Net().world);
      send[0] = static_cast<int32_t>(local.size());
      std::copy(local.begin(), local.end(), send.begin() + 1);
      DevBuf<int32_t> d_send, d_recv;
      d_send.Alloc(stride); d_recv.Alloc(recv.size());
      d_send.Upload(send.data(), stride, stream_);
      Net().AllGather(d_send.p, d_recv.p, stride * sizeof(int32_t), stream_);
      d_recv.Download(recv.data(), recv.size(), stream_);
      B200_CUDA(cudaStreamSynchronize(stream_));
      local.clear();
      for (int r = 0; r < Net().world; ++r) local.insert(local.end(), recv.begin() + r * stride + 1, recv.begin() + r * stride + 1 + recv[r * stride]);
      std::sort(local.begin(), local.end());
      local.erase(std::unique(local.begin(), local.end()), local.end());
    }
    if (!has) return;
    pos_values_ = local;
    const int P = static_cast<int>(pos_values_.size());
    DevBuf<int32_t> d_values;
    d_values.Alloc(P); d_values.Upload(pos_values_.data(), P, stream_);
    pos_id_.Alloc(n);
    if (n > 0) k_position_ids<<<std::max(1, std::min((n + 255) / 256, DeviceSMs() * 8)), 256, 0, stream_>>>(train_.d_position.p, n, d_values.p, P, pos_id_.p);
    B200_CUDA(cudaGetLastError());
    pos_bias_.Alloc(P); pos_bias_.Zero(stream_);
    pos_sums_.Alloc(3 * static_cast<size_t>(P));
    pos_ctrl_.Alloc(1); pos_ctrl_.Zero(stream_);
    if (P <= kRefitSharedLeaves)
      B200_CUDA(cudaFuncSetAttribute(k_refit_leaf_sums<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(3 * kRefitSharedLeaves * sizeof(long long))));
    B200_CUDA(cudaStreamSynchronize(stream_));
  }

  // After a training pass's gradients, on the stream and without a host wait: the fixed-point exponents of max|g| and max|h| over every
  // rank's rows, the per-position sums of g, h and rows (k_refit_leaf_sums with rows mapped to position ids, exact and order-free, then
  // all-reduced), and one Newton step per factor.  learning_rate and the regularisation are read from the current config.
  void UpdatePositionBias(const float* g, const float* h, int num_sms) const {
    const int n = train_.num_data, P = static_cast<int>(pos_values_.size());
    const bool net = Net().active && Net().world > 1;
    B200_CUDA(cudaMemsetAsync(&pos_ctrl_.p->absmax_bits[0], 0, 8, stream_));
    k_absmax<<<num_sms * 8, 256, 0, stream_>>>(g, h, n, pos_ctrl_.p);
    if (net) Net().AllReduce(&pos_ctrl_.p->absmax_bits[0], 2, ncclUint32, ncclMax, stream_);
    k_set_scale<<<1, 1, 0, stream_>>>(pos_ctrl_.p, 0, 1.0);
    B200_CUDA(cudaMemsetAsync(pos_sums_.p, 0, pos_sums_.n * sizeof(long long), stream_));
    if (P <= kRefitSharedLeaves)
      k_refit_leaf_sums<true><<<num_sms * 4, 256, 3 * static_cast<size_t>(P) * sizeof(long long), stream_>>>(pos_id_.p, g, h, n, P, 0, pos_ctrl_.p,
                                                                                                              pos_sums_.p);
    else
      k_refit_leaf_sums<false><<<num_sms * 8, 256, 0, stream_>>>(pos_id_.p, g, h, n, P, 0, pos_ctrl_.p, pos_sums_.p);
    if (net) Net().AllReduce(pos_sums_.p, pos_sums_.n, ncclInt64, ncclSum, stream_);
    k_position_bias_update<<<(P + 127) / 128, 128, 0, stream_>>>(pos_sums_.p, P, pos_ctrl_.p, cfg_.learning_rate,
                                                                 cfg_.lambdarank_position_bias_regularization, pos_bias_.p);
    B200_CUDA(cudaGetLastError());
  }

  const Config& cfg_;
  const Dataset& train_;
  const ObjectiveKind kind_;
  int K_ = 1;                               // trees per iteration
  double renew_alpha_ = 0.5;                // RenewAlpha
  cudaStream_t stream_ = nullptr;
  std::vector<uint8_t> need_train_;         // [K] NeedTrain, also the device table of multiclassova
  double binary_w_[2] = {1.0, 1.0};         // binary {w_neg, w_pos}
  std::vector<double> class_init_probs_;    // multiclass: [K] global class priors, then the total weight
  DevBuf<double> ova_w_; DevBuf<uint8_t> ova_need_;      // multiclassova: [K][2] {w_neg, w_pos} and need_train_ on the device
  std::vector<float> label_weight_host_; DevBuf<float> label_weight_;      // mape: 1 / max(1, |label|) (* weight)
  DevBuf<double> lr_inv_max_dcg_, lr_label_gain_, lr_discount_;      // lambdarank
  DevBuf<float> lr_sig_table_;
  double lr_min_in_ = -50, lr_max_in_ = 50, lr_idx_factor_ = 0; int lr_max_q_ = 0;
  DevBuf<unsigned> xe_state_, xe_jump_; DevBuf<double> xe_scratch_; int xe_max_q_ = 1;      // rank_xendcg: LCG per query, jump table, [2][n] rho / params
  // ranking with a position field: the sorted distinct values (global), every row's id into them, the factors, the update's sums and scales
  std::vector<int32_t> pos_values_;
  DevBuf<int> pos_id_; DevBuf<double> pos_bias_; DevBuf<long long> pos_sums_; DevBuf<TreeCtrl> pos_ctrl_;
};

}  // namespace b200gbm
