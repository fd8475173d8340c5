"""NumPy restatement of LightGBM 3.2's per-node feature sampling (`feature_fraction_bynode`) on top of interaction_ref.py (whose tree
growth grow_tree follows, with the node sample and the max_depth rule added), used to pin
the engine's device sampler (kernels.cuh d_bynode_sample) and the pick step's node filter tree by tree.

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

import numpy as np

import extra_trees_ref as X3
import interaction_ref as I
import monotone_ref as M
import split_scan_ref as ref


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


def grow_tree(bins, g, h, features, p, num_leaves, sampler, constraints=None, extra_trees=False, extra_seed=6, streams=None, mono=None,
              penalty=0.0, max_depth=-1):
    """one tree: the sampler's tree draw, then interaction_ref.grow_tree's growth (with extra_trees and, with a `mono` list, monotone
    constraints as there) where each leaf's best split is chosen among its node sample, and where a round whose left leaf is at
    `max_depth` (> 0) does not run, as the engine's round controller decides.  constraints None: unconstrained, grown as one set of every
    feature, which test_interaction_reference_cpu.py shows grows the unconstrained tree.  T["node_rounds"]: per round that ran, one
    (mask, sample) per leaf in scan order (smaller first); T["draws"]: the ColSampler draws of the tree, its tree draw included."""
    before = sampler.rnd.draws
    used = sampler.by_tree()
    constrained = constraints is not None
    cons = constraints if constrained else [[f.real_index for f in features]]
    features = sorted(features, key=lambda f: f.real_index)
    if extra_trees and streams is None:
        streams = X3.Streams(features, extra_seed)
    if not extra_trees:
        streams = None
    sets = I.sets_of(cons, max(f.real_index for f in features) + 1)
    n = len(g)
    by_real = {f.real_index: f for f in features}
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags={f.real_index: f.real_index in used for f in features}, bounds=(-math.inf, math.inf), depth=0, mask=I.ALL,
                   branch=())]
    T = dict(split_feature=[], threshold_bin=[], default_left=[], is_cat=[], cat_bins=[], split_gain=[], left_child=[], right_child=[],
             internal_value=[], internal_weight=[], internal_count=[])
    parent_of = [-1]
    rounds, picks, node_rounds = [], [], []
    new_leaves = [0]
    while True:
        counts = [leaves[l]["count"] for l in new_leaves]
        go = len(leaves) < num_leaves and not all(c < p.min_data_in_leaf * 2 for c in counts)
        if go and max_depth > 0 and leaves[new_leaves[0]]["depth"] >= max_depth:
            go = False
        if go:
            if len(new_leaves) == 2 and not counts[0] < counts[1]:
                new_leaves = new_leaves[::-1]            # smaller first (the extra-trees and the by-node draw order)
            rnd, samples = [], []
            for l in new_leaves:
                L = leaves[l]
                if mono is not None:
                    scans = M.scan_leaf(bins, g, h, L["rows"], L, features, p, mono, penalty, streams, used)
                elif streams is not None:
                    scans = X3.scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"], p, streams, used)
                else:
                    scans = ref.scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"], p)
                for fi, sc in scans.items():
                    L["flags"][fi] = sc.splittable
                allowed = {f for f in sampler.tree if sets[f] & L["mask"]} if constrained else None
                sample = sampler.by_node(allowed)
                samples.append((L["mask"], sample))
                L["best"] = I.best_of_leaf({fi: sc for fi, sc in scans.items() if fi in sample}, sets, L["mask"])
                rnd.append((l, L, scans))
            rounds.append(rnd)
            node_rounds.append(samples)
        else:
            for l in new_leaves:
                leaves[l]["best"] = None
        if len(leaves) >= num_leaves:
            break
        picks.append([(li, L["best"]) for li, L in enumerate(leaves) if L["best"] is not None])
        pick = None
        for li, L in enumerate(leaves):
            b = L["best"]
            if b is not None and (pick is None or ref.better_split(b.gain, b.feature, leaves[pick]["best"].gain, leaves[pick]["best"].feature)):
                pick = li
        if pick is None or not leaves[pick]["best"].gain > 0.0:
            break
        L, sp = leaves[pick], leaves[pick]["best"]
        f = by_real[sp.feature]
        left = ref.goes_left(bins[L["rows"], f.real_index].astype(np.int64), f, sp)
        sum_h2 = L["sum_h"] + 2 * ref.K_EPS
        if mono is not None:
            lo, hi = L["bounds"]
            left_out = M.constrained_output(sp.left_g, sp.left_h, p, sp.l2, lo, hi)
            right_out = M.constrained_output(L["sum_g"] - sp.left_g, sum_h2 - sp.left_h, p, sp.l2, lo, hi)
            lb, rb = M.child_bounds(L["bounds"], 0 if sp.is_cat else mono[sp.feature], sp.is_cat, left_out, right_out)
        else:
            left_out = ref.calc_output(sp.left_g, sp.left_h, p, sp.l2)
            right_out = ref.calc_output(L["sum_g"] - sp.left_g, sum_h2 - sp.left_h, p, sp.l2)
            lb = rb = L["bounds"]
        mask, branch = L["mask"] & sets[sp.feature], L["branch"] + (sp.feature,)
        node, nl = len(leaves) - 1, len(leaves)
        par = parent_of[pick]
        if par >= 0:
            if T["left_child"][par] == ~pick:
                T["left_child"][par] = node
            else:
                T["right_child"][par] = node
        T["split_feature"].append(sp.feature); T["threshold_bin"].append(0 if sp.is_cat else sp.threshold)
        T["default_left"].append(bool(sp.default_left)); T["is_cat"].append(sp.is_cat); T["cat_bins"].append(sp.cat_bins)
        T["split_gain"].append(float(np.float32(sp.gain + p.min_gain_to_split)))
        T["left_child"].append(~pick); T["right_child"].append(~nl)
        T["internal_value"].append(L["value"]); T["internal_weight"].append(L["weight"]); T["internal_count"].append(L["count"])
        lrows, rrows = L["rows"][left], L["rows"][~left]
        flags = dict(L["flags"])
        R = dict(rows=rrows, sum_g=L["sum_g"] - sp.left_g, sum_h=sum_h2 - sp.left_h - ref.K_EPS, count=len(rrows), best=None,
                 value=0.0 if math.isnan(right_out) else right_out, weight=sum_h2 - sp.left_h - ref.K_EPS, flags=dict(flags), bounds=rb,
                 depth=L["depth"] + 1, mask=mask, branch=branch)
        L.update(rows=lrows, sum_g=sp.left_g, sum_h=sp.left_h - ref.K_EPS, count=len(lrows), best=None,
                 value=0.0 if math.isnan(left_out) else left_out, weight=sp.left_h - ref.K_EPS, flags=flags, bounds=lb, depth=L["depth"] + 1,
                 mask=mask, branch=branch)
        leaves.append(R)
        parent_of[pick] = node
        parent_of.append(node)
        new_leaves = [pick, nl]
    T["num_leaves"] = len(leaves)
    T["leaf_value"] = [L["value"] if abs(L["value"]) > ref.K_ZERO else 0.0 for L in leaves]
    T["leaf_weight"] = [L["weight"] for L in leaves]
    T["leaf_count"] = [L["count"] for L in leaves]
    T["internal_value"] = [v if abs(v) > ref.K_ZERO else 0.0 for v in T["internal_value"]]
    T["masks"] = [L["mask"] for L in leaves]
    T["branches"] = [L["branch"] for L in leaves]
    T["rounds"], T["picks"], T["scanned_counts"] = rounds, picks, []
    T["node_rounds"] = node_rounds
    T["draws"] = sampler.rnd.draws - before
    return T
