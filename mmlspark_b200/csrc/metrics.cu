// Metrics (metrics.h).  Included by engine.cu; only the reduced sums of the metric kernels cross PCIe.
#include "metrics.h"
#include "objective.h"

namespace b200gbm {

const Metrics::Info Metrics::kInfos[] = {
    {"l2", kPointwise, kMetL2}, {"rmse", kPointwise, kMetL2, kNoCheck, true}, {"l1", kPointwise, kMetL1}, {"huber", kPointwise, kMetHuber},
    {"fair", kPointwise, kMetFair}, {"poisson", kPointwise, kMetPoisson}, {"gamma", kPointwise, kMetGamma},
    {"gamma_deviance", kPointwise, kMetGammaDeviance}, {"tweedie", kPointwise, kMetTweedie}, {"quantile", kPointwise, kMetQuantile},
    {"mape", kPointwise, kMetMape}, {"binary_logloss", kPointwise, kMetBinLogloss}, {"binary_error", kPointwise, kMetBinError},
    {"multi_logloss", kPointwise, kMetMultiLogloss, kMultiOutput}, {"multi_error", kPointwise, kMetMultiError, kMultiOutput},
    {"cross_entropy", kPointwise, kMetXent}, {"cross_entropy_lambda", kPointwise, kMetXentLambda, kUnitLabels},
    {"kullback_leibler", kPointwise, kMetKLDiv, kUnitLabelsWeights}, {"auc", kAuc}, {"average_precision", kAveragePrecision},
    {"auc_mu", kAucMu, 0, kClassLabels}, {"ndcg", kRank, 0}, {"map", kRank, 1}};

Metrics::Metrics(const Config& cfg, const Objective& obj, const Dataset& train)
    : obj_(obj), train_(train), K_(obj.NumTreePerIteration()), num_sms_(DeviceSMs()) { Reset(cfg, {}); met_out_.Alloc(2 * kMaxEvalAt); }

void Metrics::Reset(const Config& cfg, const std::vector<ValidSet*>& valids) {
  Plan plan = Parse(cfg);
  Check(plan, train_);
  for (const ValidSet* v : valids) Check(plan, *v->ds);
  plan_ = std::move(plan);
}

Metrics::Plan Metrics::Parse(const Config& cfg) const {
  Plan p;
  for (const std::string& m : cfg.metric) {
    const Info* info = std::find_if(std::begin(kInfos), std::end(kInfos), [&](const Info& i) { return m == i.name; });
    if (info == std::end(kInfos)) Fatal("Unknown metric type name: " + m);
    p.entries.push_back(Entry{info, {}});
    if (info->family == kRank) for (int k : cfg.eval_at) p.names.push_back(m + "@" + std::to_string(k));
    else p.names.push_back(m);
  }
  if (cfg.eval_at.size() > static_cast<size_t>(kMaxEvalAt)) Fatal("eval_at: at most " + std::to_string(kMaxEvalAt) + " positions are supported");
  HostModel::OutputTransform t; HostModel::ObjectiveTransform(obj_.ToString(), &t);
  for (Entry& e : p.entries) {
    const Info& m = *e.info;
    if (m.family == kPointwise)
      e.mp = MetricParams{m.kind, K_, obj_.kind() == ObjectiveKind::kMulticlassOva ? 1 : 0, t.kind, cfg.alpha, cfg.fair_c,
                          cfg.tweedie_variance_power, cfg.sigmoid, t.sigmoid};
    if (m.family == kRank) (m.kind == 0 ? p.rank.want_ndcg : p.rank.want_map) = 1;
    if (m.check == kClassLabels) {
      if (K_ < 2) Fatal(std::string("metric ") + m.name + " needs a multiclass objective");
      // [UPSTREAM Config::GetAucMuWeights]: the given K x K matrix or 1 off the diagonal; the diagonal is set to 0 either way
      if (!cfg.auc_mu_weights.empty() && cfg.auc_mu_weights.size() != static_cast<size_t>(K_) * K_)
        Fatal("auc_mu_weights must have " + std::to_string(K_ * K_) + " elements, but found " + std::to_string(cfg.auc_mu_weights.size()));
      std::vector<double> wm = cfg.auc_mu_weights.empty() ? std::vector<double>(static_cast<size_t>(K_) * K_, 1.0) : cfg.auc_mu_weights;
      for (int c = 0; c < K_; ++c) wm[static_cast<size_t>(c) * K_ + c] = 0.0;
      for (int i = 0; i < K_; ++i)      // the pairs (0,1), (0,2), ..., (K-2,K-1) and their rows (t1, v) of EvalAucMu
        for (int j = i + 1; j < K_; ++j) {
          p.mu_pairs.push_back(make_int2(i, j));
          std::vector<double> v(K_);
          for (int c = 0; c < K_; ++c) v[c] = wm[static_cast<size_t>(i) * K_ + c] - wm[static_cast<size_t>(j) * K_ + c];
          p.mu_pv.push_back(v[i] - v[j]);
          p.mu_pv.insert(p.mu_pv.end(), v.begin(), v.end());
        }
    }
  }
  p.rank.nk = static_cast<int>(std::copy(cfg.eval_at.begin(), cfg.eval_at.end(), p.rank.ks) - p.rank.ks);
  std::sort(p.rank.ks, p.rank.ks + p.rank.nk);
  for (int k : cfg.eval_at) p.eval_pos.push_back(static_cast<int>(std::find(p.rank.ks, p.rank.ks + p.rank.nk, k) - p.rank.ks));
  p.label_gain = LabelGain(cfg);
  return p;
}

void Metrics::Check(const Plan& plan, const Dataset& ds) const {
  for (const Entry& e : plan.entries) {
    const std::string m = e.info->name;
    if (e.info->check == kClassLabels)      // the class of a row is its label cast to int, as the multiclass objectives read it
      for (float y : ds.label) {
        const int l = static_cast<int>(y);
        if (!(y > -1.0f && y < static_cast<float>(K_)) || l < 0 || l >= K_)
          Fatal("Label must be in [0, " + std::to_string(K_) + "), but found " + std::to_string(l) + " in label");
      }
    if (e.info->check != kUnitLabels && e.info->check != kUnitLabelsWeights) continue;
    if (K_ > 1) Fatal("metric " + m + " needs a single-output objective");
    for (float y : ds.label) if (!(y >= 0.0f && y <= 1.0f)) Fatal("[" + m + "]: does not tolerate label " + std::to_string(y) + " outside [0, 1]");
    if (e.info->check == kUnitLabelsWeights && !ds.weight.empty()) {
      double sw = 0; for (float w : ds.weight) { if (w < 0) Fatal("[" + m + "]: at least one weight is negative"); sw += w; }
      if (!(sw > 0)) Fatal("[" + m + "]: sum of weights is zero");
    }
  }
}

std::vector<double> Metrics::Eval(const double* score, const Dataset& ds, cudaStream_t s) {
  const int n = ds.num_data;
  if (ds.label.empty()) Fatal("label should not be empty for evaluation");
  const float *d_y = ds.d_label.p, *d_w = ds.weight.empty() ? nullptr : ds.d_weight.p;
  const int grid = std::max(1, std::min((n + kMetricBlock - 1) / kMetricBlock, num_sms_ * 8));
  if (met_partial_.n < static_cast<size_t>(grid) * 2 * kMaxEvalAt) met_partial_.Alloc(static_cast<size_t>(grid) * 2 * kMaxEvalAt);
  std::vector<double> out;
  // averaged metrics are global in distributed mode (B.5)
  auto avg = [&](double loss, double sw) { double v[2] = {loss, sw}; AllReduceHost(v, 2, ncclSum, s); return v[0] / v[1]; };
  std::vector<double> rank_vals[2];      // ndcg, map at the eval_at positions (Config never leaves eval_at empty)
  for (const Entry& e : plan_.entries) {
    const Info& m = *e.info;
    if (m.family == kPointwise) {
      if (m.check == kMultiOutput && K_ < 2) Fatal(std::string("metric ") + m.name + " needs a multiclass objective");
      k_metric_pointwise<<<grid, kMetricBlock, 0, s>>>(score, d_y, d_w, n, e.mp, met_partial_.p);
      k_metric_finish<<<1, 32, 0, s>>>(met_partial_.p, grid, 2, met_out_.p);
      B200_CUDA(cudaGetLastError());
      double v[2]; Fetch(v, 2, s);
      const double a = avg(v[0], v[1]);
      out.push_back(m.root ? std::sqrt(a) : a);
    } else if (m.family == kAuc || m.family == kAveragePrecision) {
      // [UPSTREAM AUCMetric::Eval / AveragePrecisionMetric::Eval] are rank-local (no network sync): sort by descending score, then the
      // prefix sums of the split weights and the tie groups' starts
      if (auc_keys_a_.n < static_cast<size_t>(n)) {
        auc_keys_a_.Alloc(n); auc_keys_b_.Alloc(n); auc_rows_a_.Alloc(n); auc_rows_b_.Alloc(n); auc_wpos_.Alloc(n); auc_wneg_.Alloc(n);
        auc_ppos_.Alloc(n); auc_pneg_.Alloc(n); auc_head_.Alloc(n); auc_start_.Alloc(n);
        size_t t1 = 0, t2 = 0, t3 = 0;
        cub::DeviceRadixSort::SortPairsDescending(nullptr, t1, auc_keys_a_.p, auc_keys_b_.p, auc_rows_a_.p, auc_rows_b_.p, n, 0, 64, s);
        cub::DeviceScan::InclusiveSum(nullptr, t2, auc_wpos_.p, auc_ppos_.p, n, s);
        cub::DeviceScan::InclusiveScan(nullptr, t3, auc_head_.p, auc_start_.p, cub::Max(), n, s);
        auc_tmp_.Alloc(std::max(t1, std::max(t2, t3)) + 16);
      }
      size_t tb = auc_tmp_.n;
      k_auc_keys<<<num_sms_ * 8, 256, 0, s>>>(score, n, auc_keys_a_.p, auc_rows_a_.p);
      B200_CUDA(cub::DeviceRadixSort::SortPairsDescending(auc_tmp_.p, tb, auc_keys_a_.p, auc_keys_b_.p, auc_rows_a_.p, auc_rows_b_.p, n, 0, 64, s));
      k_auc_weights<<<num_sms_ * 8, 256, 0, s>>>(auc_keys_b_.p, auc_rows_b_.p, d_y, d_w, n, auc_wpos_.p, auc_wneg_.p, auc_head_.p);
      tb = auc_tmp_.n; B200_CUDA(cub::DeviceScan::InclusiveSum(auc_tmp_.p, tb, auc_wpos_.p, auc_ppos_.p, n, s));
      tb = auc_tmp_.n; B200_CUDA(cub::DeviceScan::InclusiveSum(auc_tmp_.p, tb, auc_wneg_.p, auc_pneg_.p, n, s));
      tb = auc_tmp_.n; B200_CUDA(cub::DeviceScan::InclusiveScan(auc_tmp_.p, tb, auc_head_.p, auc_start_.p, cub::Max(), n, s));
      const bool auc = m.family == kAuc;
      if (auc) k_auc_terms<<<grid, kMetricBlock, 0, s>>>(auc_keys_b_.p, auc_start_.p, auc_ppos_.p, auc_pneg_.p, n, met_partial_.p);
      else k_ap_terms<<<grid, kMetricBlock, 0, s>>>(auc_keys_b_.p, auc_start_.p, auc_ppos_.p, auc_pneg_.p, n, met_partial_.p);
      k_metric_finish<<<1, 32, 0, s>>>(met_partial_.p, grid, 2, met_out_.p);
      B200_CUDA(cudaGetLastError());
      double v[2], tot[2];
      B200_CUDA(cudaMemcpyAsync(&tot[0], auc_ppos_.p + (n - 1), sizeof(double), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaMemcpyAsync(&tot[1], auc_pneg_.p + (n - 1), sizeof(double), cudaMemcpyDeviceToHost, s));
      Fetch(v, 2, s);      // synchronises the stream, so tot has arrived as well
      // a single-class set scores 1 ([UPSTREAM] sum_pos > 0 && sum_pos != sum_weights for average_precision)
      out.push_back(!(tot[0] > 0 && tot[1] > 0) ? 1.0 : auc ? v[0] / (tot[0] * tot[1]) : v[0] / tot[0]);
    } else if (m.family == kAucMu) {
      out.push_back(EvalAucMu(score, d_y, d_w, n, s));      // [UPSTREAM AucMuMetric::Eval] rank-local as well
    } else {      // ndcg and map come from one launch of the rank kernel
      if (rank_vals[0].empty()) {
        const int nq = static_cast<int>(ds.query_boundaries.size()) - 1;
        if (nq <= 0) Fatal(std::string("The ") + (m.kind == 0 ? "NDCG" : "MAP") + " metric requires query information");
        int max_q = 1; for (int q = 0; q < nq; ++q) max_q = std::max(max_q, ds.query_boundaries[q + 1] - ds.query_boundaries[q]);
        const std::vector<double> disc = DcgDiscount(max_q);
        DevBuf<double> d_lg, d_disc;
        d_lg.Alloc(plan_.label_gain.size()); d_lg.Upload(plan_.label_gain.data(), plan_.label_gain.size(), s);
        d_disc.Alloc(disc.size()); d_disc.Upload(disc.data(), disc.size(), s);
        const size_t smem = static_cast<size_t>(max_q) * (8 + 4 + 4);
        if (smem > 200 * 1024) Fatal("a query group is too large for the ranking metric kernel");
        B200_CUDA(cudaFuncSetAttribute(k_metric_rank, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(std::max<size_t>(smem, 1024))));
        const int rgrid = std::max(1, std::min(nq, num_sms_ * 8));
        if (met_partial_.n < static_cast<size_t>(rgrid) * 2 * kMaxEvalAt) met_partial_.Alloc(static_cast<size_t>(rgrid) * 2 * kMaxEvalAt);
        k_metric_rank<<<rgrid, 128, std::max<size_t>(smem, 1024), s>>>(score, d_y, ds.d_qb.p, nq, d_lg.p, static_cast<int>(plan_.label_gain.size()), d_disc.p, plan_.rank, max_q, met_partial_.p);
        k_metric_finish<<<1, 32, 0, s>>>(met_partial_.p, rgrid, 2 * kMaxEvalAt, met_out_.p);
        B200_CUDA(cudaGetLastError());
        double v[2 * kMaxEvalAt]; Fetch(v, 2 * kMaxEvalAt, s);
        for (int pos : plan_.eval_pos) {
          rank_vals[0].push_back(avg(v[pos], nq));
          rank_vals[1].push_back(avg(v[kMaxEvalAt + pos], nq));
        }
      }
      out.insert(out.end(), rank_vals[m.kind].begin(), rank_vals[m.kind].end());
    }
  }
  return out;
}

// [UPSTREAM AucMuMetric::Eval]: for each class pair i < j, the weighted AUC of class i against class j ranked by
// d = t1 * (Wm[i,:] - Wm[j,:]) . s, t1 = v[i] - v[j]; auc_mu is the mean over the pairs.  Pairs run in batches of consecutive pairs
// whose segments (the rows of both classes) hold at most about 2n items, so the scratch is O(n) however many classes there are.
double Metrics::EvalAucMu(const double* score, const float* d_y, const float* d_w, int n, cudaStream_t s) {
  const int eg = num_sms_ * 8;
  // the class-grouped row order and the class boundaries
  const size_t m = static_cast<size_t>(std::max(n, 1));
  if (mu_cls_keys_a_.n < m) { mu_cls_keys_a_.Alloc(m); mu_cls_keys_b_.Alloc(m); mu_cls_rows_a_.Alloc(m); mu_cls_rows_b_.Alloc(m); }
  if (mu_cls_start_.n < static_cast<size_t>(K_) + 1) mu_cls_start_.Alloc(K_ + 1);
  int bits = 1; while ((1 << bits) < K_) ++bits;
  auto ensure_tmp = [&](size_t bytes) { if (mu_tmp_.n < bytes) mu_tmp_.Alloc(bytes + 16); };
  size_t tb = 0;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, mu_cls_keys_a_.p, mu_cls_keys_b_.p, mu_cls_rows_a_.p, mu_cls_rows_b_.p, n, 0, bits, s));
  ensure_tmp(tb);
  mu_cls_start_.Zero(s);
  if (n > 0) {
    k_class_keys<<<eg, 256, 0, s>>>(d_y, n, mu_cls_keys_a_.p, mu_cls_rows_a_.p);
    tb = mu_tmp_.n;
    B200_CUDA(cub::DeviceRadixSort::SortPairs(mu_tmp_.p, tb, mu_cls_keys_a_.p, mu_cls_keys_b_.p, mu_cls_rows_a_.p, mu_cls_rows_b_.p, n, 0, bits, s));
    k_class_bounds<<<eg, 256, 0, s>>>(mu_cls_keys_b_.p, n, K_, mu_cls_start_.p);
  }
  std::vector<int> cls_start(K_ + 1);
  mu_cls_start_.Download(cls_start.data(), K_ + 1, s);
  B200_CUDA(cudaStreamSynchronize(s));
  const std::vector<int2>& pairs = plan_.mu_pairs;
  const std::vector<double>& pv = plan_.mu_pv;
  const int npairs = static_cast<int>(pairs.size());
  // a batch closes before it passes cap items (one oversized pair still makes a batch of its own) or kMaxPairs pairs, which bounds the
  // per-block partials; item offsets inside a batch stay below 2^31
  const long long cap = std::max<long long>(1, std::min<long long>(2LL * n, 1LL << 30));
  constexpr int kMaxPairs = 1024;
  // cub's segmented sort gives a large segment one thread block, so a segment of at least kLargeSegment items is sorted by a
  // device-wide radix sort of its own instead and is left out of the segmented sort (its end offset there equals its begin)
  constexpr int kLargeSegment = 1 << 16;
  // batch b: pairs [batch_first[b], batch_first[b + 1]), their offsets and segmented-sort ends at offs[off_base[b]], ends_small[off_base[b]]
  std::vector<int> batch_first, off_base, offs, ends_small;
  long long items = 0, max_items = 0; int max_pairs = 0;
  for (int p = 0; p < npairs; ++p) {
    const long long sz = (cls_start[pairs[p].x + 1] - cls_start[pairs[p].x]) + (cls_start[pairs[p].y + 1] - cls_start[pairs[p].y]);
    const bool open = !batch_first.empty() && p - batch_first.back() < kMaxPairs && items + sz <= cap;
    if (!open) {
      if (!batch_first.empty()) { offs.push_back(static_cast<int>(items)); ends_small.push_back(0); }
      batch_first.push_back(p); off_base.push_back(static_cast<int>(offs.size())); items = 0;
    }
    offs.push_back(static_cast<int>(items));
    ends_small.push_back(static_cast<int>(sz >= kLargeSegment ? items : items + sz));
    items += sz;
    max_items = std::max(max_items, items);
    max_pairs = std::max(max_pairs, p - batch_first.back() + 1);
  }
  offs.push_back(static_cast<int>(items)); ends_small.push_back(0);
  batch_first.push_back(npairs);
  const int nb = static_cast<int>(off_base.size());
  const size_t mi = static_cast<size_t>(std::max<long long>(max_items, 1));
  if (mu_keys_a_.n < mi) {
    mu_keys_a_.Alloc(mi); mu_keys_b_.Alloc(mi); mu_rows_a_.Alloc(mi); mu_rows_b_.Alloc(mi); mu_seg_.Alloc(mi); mu_head_.Alloc(mi);
    mu_start_.Alloc(mi); mu_wpos_.Alloc(mi); mu_wneg_.Alloc(mi); mu_ppos_.Alloc(mi); mu_pneg_.Alloc(mi);
  }
  if (mu_pairs_.n < pairs.size()) mu_pairs_.Alloc(pairs.size());
  if (mu_pv_.n < pv.size()) mu_pv_.Alloc(pv.size());
  if (mu_off_.n < offs.size()) { mu_off_.Alloc(offs.size()); mu_end_small_.Alloc(offs.size()); }
  if (mu_pair_auc_.n < static_cast<size_t>(npairs)) mu_pair_auc_.Alloc(npairs);
  if (mu_partial_.n < static_cast<size_t>(eg) * max_pairs) mu_partial_.Alloc(static_cast<size_t>(eg) * max_pairs);
  mu_pairs_.Upload(pairs.data(), pairs.size(), s);
  mu_pv_.Upload(pv.data(), pv.size(), s);
  mu_off_.Upload(offs.data(), offs.size(), s);
  mu_end_small_.Upload(ends_small.data(), ends_small.size(), s);
  for (int b = 0; b < nb; ++b) {
    const int p0 = batch_first[b], P = batch_first[b + 1] - p0;
    const int* off = mu_off_.p + off_base[b];
    const int* end_small = mu_end_small_.p + off_base[b];
    const int* hoff = offs.data() + off_base[b];
    const int N = hoff[P];
    if (N > 0) {
      k_aucmu_keys<<<eg, 256, 0, s>>>(score, n, K_, mu_cls_start_.p, mu_cls_rows_b_.p, mu_pairs_.p, mu_pv_.p, p0, P, off, mu_keys_a_.p, mu_rows_a_.p, mu_seg_.p);
      size_t t1 = 0, t2 = 0, t3 = 0, t4 = 0; int largest = 0;
      for (int g = 0; g < P; ++g) largest = std::max(largest, hoff[g + 1] - hoff[g]);
      B200_CUDA(cub::DeviceSegmentedSort::StableSortPairsDescending(nullptr, t1, mu_keys_a_.p, mu_keys_b_.p, mu_rows_a_.p, mu_rows_b_.p, N, P, off, end_small, s));
      B200_CUDA(cub::DeviceScan::InclusiveSumByKey(nullptr, t2, mu_seg_.p, mu_wpos_.p, mu_ppos_.p, N, cuda::std::equal_to<>(), s));
      B200_CUDA(cub::DeviceScan::InclusiveScan(nullptr, t3, mu_head_.p, mu_start_.p, cub::Max(), N, s));
      B200_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, t4, mu_keys_a_.p, mu_keys_b_.p, mu_rows_a_.p, mu_rows_b_.p, largest, 0, 64, s));
      ensure_tmp(std::max(std::max(t1, t2), std::max(t3, t4)));
      tb = mu_tmp_.n;
      B200_CUDA(cub::DeviceSegmentedSort::StableSortPairsDescending(mu_tmp_.p, tb, mu_keys_a_.p, mu_keys_b_.p, mu_rows_a_.p, mu_rows_b_.p, N, P, off, end_small, s));
      for (int g = 0; g < P; ++g) {      // the large segments (radix sorts are stable, as the segmented sort is)
        const int o = hoff[g], len = hoff[g + 1] - o;
        if (len < kLargeSegment) continue;
        tb = mu_tmp_.n;
        B200_CUDA(cub::DeviceRadixSort::SortPairsDescending(mu_tmp_.p, tb, mu_keys_a_.p + o, mu_keys_b_.p + o, mu_rows_a_.p + o, mu_rows_b_.p + o, len, 0, 64, s));
      }
      k_aucmu_weights<<<eg, 256, 0, s>>>(mu_keys_b_.p, mu_rows_b_.p, mu_seg_.p, off, mu_pairs_.p, p0, d_y, d_w, N, mu_wpos_.p, mu_wneg_.p, mu_head_.p);
      tb = mu_tmp_.n; B200_CUDA(cub::DeviceScan::InclusiveSumByKey(mu_tmp_.p, tb, mu_seg_.p, mu_wpos_.p, mu_ppos_.p, N, cuda::std::equal_to<>(), s));
      tb = mu_tmp_.n; B200_CUDA(cub::DeviceScan::InclusiveSumByKey(mu_tmp_.p, tb, mu_seg_.p, mu_wneg_.p, mu_pneg_.p, N, cuda::std::equal_to<>(), s));
      tb = mu_tmp_.n; B200_CUDA(cub::DeviceScan::InclusiveScan(mu_tmp_.p, tb, mu_head_.p, mu_start_.p, cub::Max(), N, s));
    }
    B200_CUDA(cudaMemsetAsync(mu_partial_.p, 0, static_cast<size_t>(eg) * P * sizeof(double), s));
    if (N > 0) k_aucmu_terms<<<eg, kMetricBlock, 0, s>>>(mu_keys_b_.p, mu_start_.p, mu_ppos_.p, mu_pneg_.p, off, P, mu_partial_.p);
    k_aucmu_pair_finish<<<(P + 127) / 128, 128, 0, s>>>(mu_partial_.p, eg, P, off, mu_ppos_.p, mu_pneg_.p, p0, mu_pair_auc_.p);
    B200_CUDA(cudaGetLastError());
  }
  k_aucmu_total<<<1, 32, 0, s>>>(mu_pair_auc_.p, npairs, K_, met_out_.p);
  B200_CUDA(cudaGetLastError());
  double v = 0; Fetch(&v, 1, s);
  return v;
}

}  // namespace b200gbm
