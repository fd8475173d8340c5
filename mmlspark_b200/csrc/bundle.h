// Exclusive feature bundling: which sparse features share one uint8 storage column.
//
// LightGBM bundles features that are rarely non-zero together (enable_bundle, on by default) and tolerates a few conflicting rows.  This
// engine keeps a bundle only if NO row of the dataset has two of its members away from their most frequent bin (mfb): the grouping below
// is drawn on the bin-construction sample, and every row is then checked on the device (k_bundle_conflicts*, kernels.cuh) before any bin
// is written; a bundle with a conflicting row is dissolved.  Under that rule a member's histogram is rebuilt exactly from its column
// (d_unbundle_hist), so models are identical to unbundled training.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "bin_mapper.h"

namespace b200gbm {

// non-trivial numerical uint8 features whose most frequent bin is the bin of zero
inline bool BundleCandidate(const FeatureBins& fb) {
  return !fb.trivial && !fb.categorical && fb.num_bin <= 256 && fb.most_freq_bin == fb.default_bin;
}

// Greedy, deterministic grouping.  off_mfb[f] = the ascending sampled rows (< sample_cnt) in which candidate f is away from its mfb.
// Candidates are visited by descending count of such rows (ties: lower real index first); each joins the first bundle, in creation order
// among the kSearchBundles most recently opened ones, that shares none of its sampled rows and stays within 256 slots (slot 0 = all
// members at their mfb, each member adds num_bin - 1), else it opens a new bundle.  The window bounds the work per candidate and the
// memory (one sample-row bitmap per bundle in the window) on wide data whose candidates mostly conflict, where every candidate opens a
// bundle of its own ([UPSTREAM] FindGroups likewise searches at most max_search_group = 100 groups).
// Returns the bundles of two or more members (real indices, in joining order).
constexpr int kSearchBundles = 100;
inline std::vector<std::vector<int>> FindBundles(const std::vector<FeatureBins>& mappers, const std::vector<std::vector<int>>& off_mfb,
                                                 int sample_cnt) {
  std::vector<int> cand;
  for (int f = 0; f < static_cast<int>(mappers.size()); ++f)
    if (BundleCandidate(mappers[f])) cand.push_back(f);
  std::stable_sort(cand.begin(), cand.end(), [&](int a, int b) { return off_mfb[a].size() > off_mfb[b].size(); });
  struct Group {
    std::vector<int> members;
    std::vector<uint64_t> rows;      // bitmap of the sampled rows some member is away from its mfb in (freed once out of the window)
    int slots = 1;
    size_t nrows = 0;                // set bits of `rows`
  };
  std::vector<Group> groups;
  const size_t words = (static_cast<size_t>(std::max(sample_cnt, 0)) + 63) / 64;
  for (int f : cand) {
    const int need = mappers[f].num_bin - 1;
    const std::vector<int>& rows = off_mfb[f];
    Group* g = nullptr;
    for (size_t k = groups.size() > kSearchBundles ? groups.size() - kSearchBundles : 0; k < groups.size(); ++k) {
      Group& gi = groups[k];
      if (gi.slots + need > 256 || gi.nrows + rows.size() > static_cast<size_t>(sample_cnt)) continue;      // no room, or rows must overlap
      bool clash = false;
      for (int r : rows) if ((gi.rows[r >> 6] >> (r & 63)) & 1u) { clash = true; break; }
      if (!clash) { g = &gi; break; }
    }
    if (!g) {
      if (groups.size() >= kSearchBundles) std::vector<uint64_t>().swap(groups[groups.size() - kSearchBundles].rows);      // leaves the window
      groups.emplace_back();
      g = &groups.back();
      g->rows.assign(words, 0);
    }
    g->members.push_back(f);
    g->slots += need;
    g->nrows += rows.size();
    for (int r : rows) g->rows[r >> 6] |= uint64_t{1} << (r & 63);
  }
  std::vector<std::vector<int>> out;
  for (Group& g : groups) if (g.members.size() >= 2) out.push_back(std::move(g.members));
  return out;
}

}  // namespace b200gbm
