// LGBM_BoosterRefit: every tree keeps its structure and each leaf value is re-estimated from the training rows the caller's leaf
// indices place in it.  Restated from LightGBM v3.2.x GBDT::RefitTree + SerialTreeLearner::FitByExistingTree (from knowledge): for each
// iteration the objective's gradients at the current training scores (every row, no bagging or GOSS sample), then per class the
// leaf rule of refit_kernels.cuh and the class's scores plus the new tree.  Validation scores are not touched.
// Differences from upstream, on purpose: the per-leaf sums are all-reduced across data-parallel ranks, so every rank ends with the one
// model of all rows (upstream refits each rank on its own rows); a negative leaf index is rejected; boosting=rf fails.
// Part of engine.cu's translation unit (refit.cu is included there).
#include "refit_kernels.cuh"

namespace b200gbm {

constexpr size_t kRefitBlockBytes = static_cast<size_t>(64) << 20;      // each of the two pinned row-block buffers
constexpr size_t kRefitReserve = static_cast<size_t>(1) << 30;          // device memory left free beside the refit's buffers

// B200GBM_REFIT_STAGING=models,rows (tests): at most that many models per batch and rows per pinned row block (0: no cap), so that small
// data goes through several batches and row blocks
struct RefitCap { long long models = 0, rows = 0; };
static RefitCap RefitStagingCap() {
  RefitCap c;
  const char* env = std::getenv("B200GBM_REFIT_STAGING");
  if (env && std::sscanf(env, "%lld,%lld", &c.models, &c.rows) < 1) c = RefitCap();
  return c;
}

void Booster::Refit(const int32_t* leaf_preds, int nrow, int ncol) {
  if (!train) Fatal("refit needs a training booster: this booster was loaded from a model string");
  EnsureDevice();
  const int n = train->num_data;
  const int M = static_cast<int>(model.trees.size());
  const double decay = cfg.refit_decay_rate;
  cudaStream_t s = stream_;
  // this rank's checks; nothing has changed when they fail
  std::string err;
  if (custom_grad_)
    err = "No object function provided (this booster was trained on custom gradients; refit takes the objective's gradients)";
  else if (is_rf_)
    err = "boosting=rf does not support refit: a random forest's refit gradients are taken at its constant average scores, which is not "
          "restated; refit a gbdt, dart or goss booster";
  else if (!(decay >= 0.0 && decay <= 1.0))
    err = "refit_decay_rate should be in [0, 1], got " + Config::Num(decay);
  else if (!leaf_preds)
    err = "refit: leaf_preds is null";
  else if (nrow != n)
    err = "refit: leaf_preds has " + std::to_string(nrow) + " rows, the training data has " + std::to_string(n);
  else if (ncol != M)
    err = "refit: leaf_preds has " + std::to_string(ncol) + " columns, the booster has " + std::to_string(M) + " models";

  // models per batch: as many leaf columns (4 n bytes each) as fit in free device memory beside the score backup, the device row block
  // and a reserve; ranks on one device share it.  Every rank takes the smallest batch of all ranks, so all run the same collectives.
  const RefitCap cap = RefitStagingCap();
  const size_t col_bytes = static_cast<size_t>(std::max(n, 1)) * sizeof(int);
  double agree[2] = {err.empty() ? 1.0 : 0.0, static_cast<double>(std::max(M, 1))};
  if (err.empty()) {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); free_b = 0; }
    const size_t fixed = static_cast<size_t>(K) * n * sizeof(double) + kRefitBlockBytes + kRefitReserve;
    size_t fit = free_b > fixed ? (free_b - fixed) / (same_device_ ? static_cast<size_t>(Net().world) : 1) / col_bytes : 0;
    if (cap.models > 0) fit = std::min(fit, static_cast<size_t>(cap.models));
    if (fit == 0) err = "refit: not enough free device memory for one model's leaf column (" + std::to_string(col_bytes) + " bytes)";
    agree[0] = err.empty() ? 1.0 : 0.0;
    agree[1] = static_cast<double>(std::min<size_t>(std::max(fit, static_cast<size_t>(1)), static_cast<size_t>(std::max(M, 1))));
  }
  if (parallel_) AllReduceHost(agree, 2, ncclMin, s);
  if (agree[0] < 1.0) Fatal(err.empty() ? "refit: another rank's leaf_preds failed the refit checks; this rank's were fine" : err);
  if (M == 0) return;
  const int mb = static_cast<int>(agree[1]);
  const int batches = (M + mb - 1) / mb;
  size_t rows_blk = std::max<size_t>(1, std::min<size_t>(static_cast<size_t>(n), kRefitBlockBytes / (sizeof(int) * mb)));
  if (cap.rows > 0) rows_blk = std::min(rows_blk, static_cast<size_t>(cap.rows));

  // every model's leaf count, old leaf values and leaf parents (derived from the child arrays), concatenated
  std::vector<int> nl(M), parent;
  std::vector<size_t> off(M + 1, 0);
  std::vector<double> old_leaf;
  int max_leaves = 1;
  for (int m = 0; m < M; ++m) {
    const HostTree& t = *model.trees[m];
    nl[m] = t.num_leaves;
    max_leaves = std::max(max_leaves, t.num_leaves);
    off[m + 1] = off[m] + t.num_leaves;
    old_leaf.insert(old_leaf.end(), t.leaf_value.begin(), t.leaf_value.begin() + t.num_leaves);
    std::vector<int> lp(t.num_leaves, -1);
    for (int i = 0; i + 1 < t.num_leaves; ++i) {
      if (t.left_child[i] < 0) lp[~t.left_child[i]] = i;
      if (t.right_child[i] < 0) lp[~t.right_child[i]] = i;
    }
    parent.insert(parent.end(), lp.begin(), lp.end());
  }
  DevBuf<int> d_nl, d_parent, cols, dblock;
  DevBuf<double> d_old, d_new, backup;
  DevBuf<unsigned long long> first_bad;
  DevBuf<TreeCtrl> ctrl;
  DevBuf<long long> sums;
  d_nl.Alloc(M); d_nl.Upload(nl.data(), M, s);
  d_parent.Alloc(parent.size()); d_parent.Upload(parent.data(), parent.size(), s);
  d_old.Alloc(old_leaf.size()); d_old.Upload(old_leaf.data(), old_leaf.size(), s);
  d_new.Alloc(old_leaf.size());
  cols.Alloc(static_cast<size_t>(mb) * n);
  dblock.Alloc(rows_blk * mb);
  first_bad.Alloc(1); ctrl.Alloc(1); ctrl.Zero(s);
  sums.Alloc(3 * static_cast<size_t>(max_leaves));
  if (batches > 1) {      // a bad index in a later batch restores the scores the earlier batches changed
    backup.Alloc(static_cast<size_t>(K) * n);
    B200_CUDA(cudaMemcpyAsync(backup.p, score_.p, backup.n * sizeof(double), cudaMemcpyDeviceToDevice, s));
  }
  B200_CUDA(cudaFuncSetAttribute(k_refit_leaf_sums<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(3 * kRefitSharedLeaves * sizeof(long long))));
  int* pinned[2] = {nullptr, nullptr};
  cudaEvent_t copied[2] = {nullptr, nullptr};
  auto release = [&]() {
    for (int b = 0; b < 2; ++b) {
      if (copied[b]) { cudaEventSynchronize(copied[b]); cudaEventDestroy(copied[b]); }
      if (pinned[b]) cudaFreeHost(pinned[b]);
    }
  };
  SplitParams sp{};
  sp.l1 = cfg.lambda_l1; sp.l2 = cfg.lambda_l2; sp.max_delta_step = cfg.max_delta_step; sp.path_smooth = cfg.path_smooth;
  const bool const_h = obj_->ConstHessian();      // no GOSS sample here: every row's hessian is the objective's
  refit_timing = RefitTiming();
  refit_timing.batches = batches;
  try {
    for (int b = 0; b < 2; ++b) {
      B200_CUDA(cudaMallocHost(reinterpret_cast<void**>(&pinned[b]), rows_blk * mb * sizeof(int)));
      B200_CUDA(cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming));
    }
    for (int batch = 0; batch < batches; ++batch) {
      const int m0 = batch * mb, m1 = std::min(M, m0 + mb), bm = m1 - m0;
      // staging: row blocks of the batch's columns through the two pinned buffers (the host fills one while the other is copied), then
      // transposed into leaf columns and range-checked on the device
      auto t0 = std::chrono::steady_clock::now();
      B200_CUDA(cudaMemsetAsync(first_bad.p, 0xff, sizeof(unsigned long long), s));
      int blk = 0;
      for (long long r0 = 0; r0 < n; r0 += static_cast<long long>(rows_blk), ++blk) {
        const int rows = static_cast<int>(std::min<long long>(static_cast<long long>(rows_blk), n - r0));
        int* pin = pinned[blk & 1];
        B200_CUDA(cudaEventSynchronize(copied[blk & 1]));
#pragma omp parallel for schedule(static)
        for (int i = 0; i < rows; ++i)
          std::memcpy(pin + static_cast<size_t>(i) * bm, leaf_preds + (r0 + i) * ncol + m0, sizeof(int) * bm);
        B200_CUDA(cudaMemcpyAsync(dblock.p, pin, static_cast<size_t>(rows) * bm * sizeof(int), cudaMemcpyHostToDevice, s));
        B200_CUDA(cudaEventRecord(copied[blk & 1], s));
        k_refit_stage<<<dim3((rows + 31) / 32, (bm + 31) / 32), dim3(32, 8), 0, s>>>(dblock.p, rows, bm, r0, n, m0, ncol, d_nl.p, cols.p,
                                                                                   first_bad.p);
        B200_CUDA(cudaGetLastError());
      }
      unsigned long long bad = 0;
      B200_CUDA(cudaMemcpyAsync(&bad, first_bad.p, sizeof(bad), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaStreamSynchronize(s));
      auto t1 = std::chrono::steady_clock::now();
      refit_timing.stage_ms += std::chrono::duration<double, std::milli>(t1 - t0).count();
      refit_timing.blocks += blk;
      if (bad != ~0ull) {
        const long long row = static_cast<long long>(bad / static_cast<unsigned long long>(ncol));
        const int m = static_cast<int>(bad % static_cast<unsigned long long>(ncol));
        err = "refit: leaf_preds[" + std::to_string(row) + "][" + std::to_string(m) + "] = " + std::to_string(leaf_preds[bad]) +
              " is outside [0, " + std::to_string(nl[m]) + "), the leaves of model " + std::to_string(m);
      }
      double ok = err.empty() ? 1.0 : 0.0;
      if (parallel_) AllReduceHost(&ok, 1, ncclMin, s);
      if (ok < 1.0) {
        if (batch > 0) {
          B200_CUDA(cudaMemcpyAsync(score_.p, backup.p, backup.n * sizeof(double), cudaMemcpyDeviceToDevice, s));
          B200_CUDA(cudaStreamSynchronize(s));
        }
        Fatal(err.empty() ? "refit: another rank's leaf_preds failed the refit checks; this rank's were fine" : err);
      }
      // per tree: the class's fixed-point exponents over every rank's rows, the per-leaf sums, the leaf rule, the class's scores
      for (int m = m0; m < m1; ++m) {
        const int k = m % K, L = nl[m];
        if (k == 0) {      // GBDT::Boosting at the start of each iteration
          grad_.Zero(s); hess_.Zero(s);      // classes the objective does not train read as 0, as in GetGradients
          ComputeGradientsAt(score_.p);
        }
        const float* g = grad_.p + static_cast<size_t>(k) * n;
        const float* h = hess_.p + static_cast<size_t>(k) * n;
        const int* leaf = cols.p + static_cast<size_t>(m - m0) * n;
        B200_CUDA(cudaMemsetAsync(&ctrl.p->absmax_bits[0], 0, 8, s));
        k_absmax<<<num_sms_ * 8, 256, 0, s>>>(g, h, n, ctrl.p);
        if (parallel_) Net().AllReduce(&ctrl.p->absmax_bits[0], 2, ncclUint32, ncclMax, s);
        k_set_scale<<<1, 1, 0, s>>>(ctrl.p, const_h ? 1 : 0, 1.0);
        B200_CUDA(cudaMemsetAsync(sums.p, 0, 3 * static_cast<size_t>(L) * sizeof(long long), s));
        if (L <= kRefitSharedLeaves)
          k_refit_leaf_sums<true><<<num_sms_ * 4, 256, 3 * static_cast<size_t>(L) * sizeof(long long), s>>>(leaf, g, h, n, L, const_h ? 1 : 0,
                                                                                                          ctrl.p, sums.p);
        else
          k_refit_leaf_sums<false><<<num_sms_ * 8, 256, 0, s>>>(leaf, g, h, n, L, const_h ? 1 : 0, ctrl.p, sums.p);
        if (parallel_) Net().AllReduce(sums.p, 3 * static_cast<size_t>(L), ncclInt64, ncclSum, s);
        k_refit_apply<<<(L + 127) / 128, 128, 0, s>>>(sums.p, L, ctrl.p, const_h ? 1 : 0, d_old.p + off[m], d_parent.p + off[m],
                                                      model.trees[m]->shrinkage, decay, sp, d_new.p + off[m]);
        k_refit_add_score<<<num_sms_ * 8, 256, 0, s>>>(leaf, d_new.p + off[m], n, score_.p + static_cast<size_t>(k) * n);
        B200_CUDA(cudaGetLastError());
        timing.launches += 6;
      }
      B200_CUDA(cudaStreamSynchronize(s));
      refit_timing.tree_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
    }
  } catch (...) {
    release();
    throw;
  }
  release();
  std::vector<double> new_leaf(old_leaf.size());
  d_new.Download(new_leaf.data(), new_leaf.size(), s);
  B200_CUDA(cudaStreamSynchronize(s));
  for (int m = 0; m < M; ++m) std::copy(new_leaf.begin() + off[m], new_leaf.begin() + off[m + 1], model.trees[m]->leaf_value.begin());
  predictor->Invalidate();
}

}  // namespace b200gbm
