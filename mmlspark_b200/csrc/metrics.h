// Evaluation metrics of a training Booster, chosen once from the config, with their checks and the device scratch of the metric kernels
// (metric_kernels.cuh).  Part of engine.cu's translation unit (metrics.cu is included there).
#pragma once
#include "engine.h"
#include "metric_kernels.cuh"

namespace b200gbm {

class Metrics {
 public:
  // parses cfg.metric (canonical names) and checks it against the objective and the training data
  Metrics(const Config& cfg, const Objective& obj, const Dataset& train);
  // the same, and every validation set, for a changed config; nothing changes unless every check passes.  The scratch is kept: the
  // estimators' learning-rate schedule resets the parameters every iteration.
  void Reset(const Config& cfg, const std::vector<ValidSet*>& valids);
  const std::vector<std::string>& Names() const { return plan_.names; }      // ndcg / map: one name per eval_at position
  void CheckData(const Dataset& ds) const { Check(plan_, ds); }      // the label and weight checks of the metrics on a dataset they evaluate
  // every metric on ds's class-major scores [K][n], in Names() order; averaged metrics are all-reduced (one AllReduceHost per value),
  // auc, average_precision and auc_mu are rank-local
  std::vector<double> Eval(const double* score, const Dataset& ds, cudaStream_t s);

 private:
  enum Family { kPointwise, kAuc, kAveragePrecision, kAucMu, kRank };
  // [UPSTREAM CrossEntropyLambdaMetric / KullbackLeiblerDivergence / AucMuMetric ::Init]; see Check, and Eval for kMultiOutput
  enum Checks { kNoCheck, kMultiOutput, kClassLabels, kUnitLabels, kUnitLabelsWeights };
  // kind: the MetricKind of a point-wise loss, or the rank kernel's output slot (0 ndcg, 1 map); root: the square root of the mean
  struct Info { const char* name; Family family; int kind = 0; Checks check = kNoCheck; bool root = false; };
  static const Info kInfos[];      // every metric the engine evaluates
  struct Entry { const Info* info; MetricParams mp; };      // mp: point-wise losses only
  struct Plan {                    // what evaluation reads from the config and the objective
    std::vector<Entry> entries;    // in cfg.metric order
    std::vector<std::string> names;
    RankEvalParams rank{};         // eval_at ascending, as the kernel evaluates it ([UPSTREAM] Config sorts eval_at) ...
    std::vector<int> eval_pos;     // ... and the position there of each eval_at in the given order, which the results keep
    std::vector<double> label_gain, mu_pv;      // mu_pv: auc_mu's row (t1, v) of each class pair in mu_pairs
    std::vector<int2> mu_pairs;
  };
  Plan Parse(const Config& cfg) const;
  void Check(const Plan& plan, const Dataset& ds) const;
  void Fetch(double* host, int count, cudaStream_t s) { met_out_.Download(host, count, s); B200_CUDA(cudaStreamSynchronize(s)); }
  double EvalAucMu(const double* score, const float* d_y, const float* d_w, int n, cudaStream_t s);

  const Objective& obj_;
  const Dataset& train_;
  const int K_, num_sms_;
  Plan plan_;
  // device scratch, grown on demand: met_* the reductions, auc_* the sort of auc / average_precision, mu_* auc_mu's class-grouped row
  // order, then one batch of class-pair segments at a time (about 2n items, so O(n) for any K)
  DevBuf<double> met_partial_, met_out_, auc_wpos_, auc_wneg_, auc_ppos_, auc_pneg_, mu_pv_, mu_wpos_, mu_wneg_, mu_ppos_, mu_pneg_, mu_partial_,
      mu_pair_auc_;
  DevBuf<unsigned long long> auc_keys_a_, auc_keys_b_, mu_keys_a_, mu_keys_b_;
  DevBuf<int> auc_rows_a_, auc_rows_b_, auc_head_, auc_start_, mu_cls_rows_a_, mu_cls_rows_b_, mu_cls_start_, mu_off_, mu_end_small_, mu_rows_a_,
      mu_rows_b_, mu_seg_, mu_head_, mu_start_;
  DevBuf<unsigned> mu_cls_keys_a_, mu_cls_keys_b_;
  DevBuf<int2> mu_pairs_;
  DevBuf<unsigned char> auc_tmp_, mu_tmp_;
};

}  // namespace b200gbm
