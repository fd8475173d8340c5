"""NumPy restatement of LightGBM 3.2's per-node feature sampling (`feature_fraction_bynode`), the rule tree_ref.grow_tree applies with a
`sampler`, used to pin the engine's device sampler (kernels.cuh d_bynode_sample) and the pick step's node filter tree by tree.

Restated from LightGBM 3.2 (ColSampler::GetByNode, ColSampler::GetCnt, SerialTreeLearner::FindBestSplitsFromHistograms); not checked
against the native library:
- One stream: ColSampler owns one Random(feature_fraction_seed).  With feature_fraction < 1 it draws the tree sample once at set-up and
  once per tree; the per-node draws continue the same stream between them.
- Every round that passes BeforeFindBestSplit (max_depth, min_data_in_leaf * 2) calls GetByNode for the smaller leaf, then for the
  larger leaf if the round has one.  No call happens after the tree stops.
- GetByNode with feature_fraction_bynode >= 1 draws nothing.  Otherwise the pool is the tree sample (every used feature without one) in
  real-index order, K = GetCnt(|pool|, feature_fraction_bynode); with interaction constraints the pool is first filtered to the
  features the leaf allows and K = min(K, |filtered|).  The sample is Random::Sample(|filtered pool|, K).
- The sample restricts only the choice of the leaf's best split: the scans, their is_splittable flags and the extra_trees draws are
  what they are without it (the filter sits where the interaction filter sits)."""
import math

import extra_trees_ref as X3


def get_cnt(total, fraction):
    """ColSampler::GetCnt"""
    return max(int(total * fraction + 0.5), min(2, total))


class CountingRandom(X3.Random):
    """Random that counts its draws"""

    def __init__(self, seed):
        super().__init__(seed)
        self.draws = 0

    def _next(self):
        self.draws += 1
        return super()._next()


def selection_branch(n, k):
    """whether Random::Sample(n, k) with 0 < k < n takes the selection branch (else Floyd's)"""
    return k > 1 and k > n / math.log2(k)


def sample_draws(n, k):
    """the draws Random::Sample(n, k) takes: n in the selection branch, k in Floyd's, none for k == n or k <= 0"""
    if k > n or k <= 0 or k == n:
        return 0
    return n if selection_branch(n, k) else k


class ColSampler:
    """one ColSampler stream over the used features (`features`, any order) for the by-tree and the by-node draws"""

    def __init__(self, features, fraction=1.0, bynode=1.0, seed=2):
        self.real = sorted(f.real_index for f in features)
        self.fraction, self.bynode = fraction, bynode
        self.rnd = CountingRandom(seed)
        self.cnt = get_cnt(len(self.real), fraction)
        self.tree = list(self.real)
        if fraction < 1.0:
            self.rnd.sample(len(self.real), self.cnt)      # the set-up draw

    def by_tree(self):
        """the next tree's feature_fraction sample (real indices, ascending)"""
        if self.fraction < 1.0:
            self.tree = [self.real[i] for i in self.rnd.sample(len(self.real), self.cnt)]
        return set(self.tree)

    def by_node(self, allowed=None):
        """GetByNode: the real indices a leaf samples; allowed: the real indices its interaction constraints allow (None: all)"""
        pool = self.tree if allowed is None else [f for f in self.tree if f in allowed]
        if self.bynode >= 1.0:
            return set(pool)
        k = min(get_cnt(len(self.tree), self.bynode), len(pool))
        return {pool[i] for i in self.rnd.sample(len(pool), k)}
