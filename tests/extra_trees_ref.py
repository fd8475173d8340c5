"""NumPy restatement of LightGBM 3.2's extremely randomised trees (`extra_trees`, `extra_seed`) on top of split_scan_ref.py, used to pin the
engine's scans (k_scan, k_scan_wide with kExtra) tree by tree and tree after tree.

Restated from LightGBM 3.2 (FeatureHistogram's USE_RAND branch, HistogramPool::SetFeatureInfo); not checked against the native library:
- Used feature i (its position among the used features in real-index order) owns Random(extra_seed + i): x = 214013 x + 2531011,
  NextInt(lo, hi) = (x & 0x7fffffff) % (hi - lo) + lo.
- Every FindBestThreshold call of the feature draws once when its range is non-empty, the smaller leaf's before the larger's.  A feature
  is scanned only in trees whose feature_fraction sample holds it and in leaves whose parent left it splittable.
- Numerical: range num_bin - 2; only the candidate with threshold == rand_threshold is evaluated in either pass (t - 1 + offset in the
  reverse pass, t + offset in the forward one), after the count and hessian tests that skip or end the pass.
- One-hot categorical: range = the num_bin - 1 category bins; only bin rand_threshold + 1 is evaluated.
- Many-vs-many categorical: range max(min(max_num_cat, used_bin) - 1, 0); only the prefixes of rand_threshold + 1 bins are evaluated,
  from either end.
- An empty range draws nothing and leaves rand_threshold at 0.

The filtered scans are taken from split_scan_ref's full scans: those record every candidate that passed the count and hessian tests
before the pass ended, which is exactly the set the random threshold is tested against."""
import math

import numpy as np

import split_scan_ref as ref


class Random:
    """LightGBM's Random (utils/random.h)"""

    def __init__(self, seed):
        self.x = seed & 0xffffffff

    def _next(self):
        self.x = (214013 * self.x + 2531011) & 0xffffffff
        return self.x

    def next_int(self, lo, hi):
        return (self._next() & 0x7fffffff) % (hi - lo) + lo

    def next_float(self):
        return ((self._next() >> 16) & 0x7fff) / 32768.0

    def sample(self, n, k):
        """Random::Sample (the engine's LcgRandom::Sample)"""
        if k > n or k <= 0:
            return []
        if k == n:
            return list(range(n))
        if k > 1 and k > n / math.log2(k):
            out = []
            for i in range(n):
                if self.next_float() < (k - len(out)) / (n - i):
                    out.append(i)
            return out
        chosen = set()
        for r in range(n - k, n):
            v = (self._next() & 0x7fffffff) % r
            chosen.add(r if v in chosen else v)
        return sorted(chosen)


def feature_fraction_sets(nf, fraction, seed, num_trees):
    """ColSampler by tree: one draw at set-up, then one per tree; the used-feature positions of every tree"""
    if fraction >= 1.0:
        return [set(range(nf))] * num_trees
    rnd = Random(seed)
    cnt = max(int(nf * fraction + 0.5), min(2, nf))
    rnd.sample(nf, cnt)
    return [set(rnd.sample(nf, cnt)) for _ in range(num_trees)]


def _counts(hh, num_bin, sum_h_in, num_data):
    cnt_factor = num_data / (sum_h_in + 2 * ref.K_EPS)
    return [ref.round_int(float(hh[b]) * cnt_factor) for b in range(num_bin)]


def numerical_range(num_bin):
    return num_bin - 2


def categorical_range(hh, num_bin, sum_h_in, num_data, p):
    if num_bin <= p.max_cat_to_onehot:
        return num_bin - 1
    cnt = _counts(hh, num_bin, sum_h_in, num_data)
    used_bin = sum(1 for b in range(1, num_bin) if cnt[b] >= p.cat_smooth)
    max_num_cat = min(p.max_cat_threshold, (used_bin + 1) // 2)
    return max(min(max_num_cat, used_bin) - 1, 0)


def _keep(r, cands):
    """r with only `cands` evaluated; returns the first strict maximum above min_gain_shift"""
    r.candidates = list(cands)
    r.splittable = any(c[0] > r.shift for c in cands)
    best = None
    for c in cands:
        if c[0] > r.shift and (best is None or c[0] > best[0]):
            best = c
    r.win = best
    r.gain = best[0] - r.shift if best is not None else ref.NEG_INF
    return best


def find_best_numerical(hg, hh, num_bin, missing_type, offset, sum_g, sum_h_in, num_data, p, feature=0, rand_threshold=None):
    r = ref.find_best_numerical(hg, hh, num_bin, missing_type, offset, sum_g, sum_h_in, num_data, p, feature)
    if rand_threshold is None:
        return r
    two_way = num_bin > 2 and missing_type == 2
    na = 1 if two_way else 0
    rev = [c for c in r.candidates if c[5] == ("rev", rand_threshold)]
    fwd = [c for c in r.candidates if c[5] == ("fwd", rand_threshold)]
    # the forward pass replaces the reverse pass's result only with a strictly larger gain: the reverse candidate comes first
    best = _keep(r, rev + fwd)
    r.threshold, r.default_left, r.left_g, r.left_h, r.left_count = 0, True, 0.0, 0.0, 0
    if best is not None:
        cnt = _counts(hh, num_bin, sum_h_in, num_data)
        t = best[5][1]
        r.threshold, r.left_g, r.left_h = t, best[1], best[2]
        if best[5][0] == "rev":
            r.left_count = num_data - sum(cnt[t + 1:num_bin - na])
        else:
            base_c = num_data - sum(cnt[1:num_bin]) if offset == 1 else 0
            r.left_count = base_c + sum(cnt[offset:t + 1])
            r.default_left = False
    if not two_way and missing_type == 2:
        r.default_left = False
    return r


def find_best_categorical(hg, hh, num_bin, sum_g, sum_h_in, num_data, p, feature=0, rand_threshold=None):
    r = ref.find_best_categorical(hg, hh, num_bin, sum_g, sum_h_in, num_data, p, feature)
    if rand_threshold is None:
        return r
    cnt = _counts(hh, num_bin, sum_h_in, num_data)
    r.cat_bins, r.left_g, r.left_h, r.left_count = (), 0.0, 0.0, 0
    if num_bin <= p.max_cat_to_onehot:
        best = _keep(r, [c for c in r.candidates if c[5] == ("onehot", rand_threshold + 1)])
        if best is not None:
            b = best[5][1]
            r.cat_bins, r.left_count = (b,), cnt[b]
    else:
        used = [b for b in range(1, num_bin) if cnt[b] >= p.cat_smooth]
        order = sorted(used, key=lambda b: (float(hg[b]) / (float(hh[b]) + p.cat_smooth), b))
        best = _keep(r, [c for c in r.candidates if c[5] in (("dir+1", rand_threshold), ("dir-1", rand_threshold))])
        if best is not None:
            seq = order if best[5][0] == "dir+1" else order[::-1]
            bins = seq[:rand_threshold + 1]
            r.cat_bins, r.left_count = tuple(sorted(bins)), sum(cnt[b] for b in bins)
    if best is not None:
        r.left_g, r.left_h = best[1], best[2]
    return r


class Streams:
    """the per-feature Random of every used feature; `features` in real-index order"""

    def __init__(self, features, extra_seed):
        self.rand = {f.real_index: Random(extra_seed + i) for i, f in enumerate(features)}

    def draw(self, f, rng):
        return self.rand[f.real_index].next_int(0, rng) if rng > 0 else 0


def scan_leaf(bins, g, h, rows, sum_g, sum_h, num_data, features, flags, p, streams, used):
    """split_scan_ref.scan_leaf with one draw per scanned feature"""
    out = {}
    for f in features:
        if f.real_index not in used or not flags[f.real_index]:
            continue
        col = bins[rows, f.real_index].astype(np.int64)
        hg = np.bincount(col, weights=g[rows], minlength=f.num_bin)
        hh = np.bincount(col, weights=h[rows], minlength=f.num_bin)
        if f.is_cat:
            t = streams.draw(f, categorical_range(hh, f.num_bin, sum_h, num_data, p))
            out[f.real_index] = find_best_categorical(hg, hh, f.num_bin, sum_g, sum_h, num_data, p, f.real_index, t)
        else:
            t = streams.draw(f, numerical_range(f.num_bin))
            out[f.real_index] = find_best_numerical(hg, hh, f.num_bin, f.missing_type, f.offset, sum_g, sum_h, num_data, p, f.real_index, t)
    return out


def grow_tree(bins, g, h, features, p, num_leaves, extra_trees=False, extra_seed=6, streams=None, used=None):
    """split_scan_ref.grow_tree with extra_trees: pass `streams` (a Streams) to carry the feature streams from tree to tree; `used`: the
    real indices the tree's feature_fraction sample holds (None: every feature).  The smaller leaf of a round (fewer rows; the right
    one on a tie) is scanned first."""
    if not extra_trees:
        return ref.grow_tree(bins, g, h, features, p, num_leaves)
    features = sorted(features, key=lambda f: f.real_index)
    if streams is None:
        streams = Streams(features, extra_seed)
    used = {f.real_index for f in features} if used is None else set(used)
    n = len(g)
    by_real = {f.real_index: f for f in features}
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags={f.real_index: f.real_index in used for f in features})]
    T = dict(split_feature=[], threshold_bin=[], default_left=[], is_cat=[], cat_bins=[], split_gain=[], left_child=[], right_child=[],
             internal_value=[], internal_weight=[], internal_count=[])
    parent_of = [-1]
    rounds, picks = [], []
    new_leaves = [0]
    while True:
        counts = [leaves[l]["count"] for l in new_leaves]
        go = len(leaves) < num_leaves and not all(c < p.min_data_in_leaf * 2 for c in counts)
        if go:
            if len(new_leaves) == 2 and not counts[0] < counts[1]:
                new_leaves = new_leaves[::-1]            # smaller first
            rnd = []
            for l in new_leaves:
                L = leaves[l]
                scans = scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"], p, streams, used)
                for fi, s in scans.items():
                    L["flags"][fi] = s.splittable
                L["best"] = ref.best_of_leaf(scans)
                rnd.append((l, L, scans))
            rounds.append(rnd)
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
        L, s = leaves[pick], leaves[pick]["best"]
        f = by_real[s.feature]
        left = ref.goes_left(bins[L["rows"], f.real_index].astype(np.int64), f, s)
        sum_h2 = L["sum_h"] + 2 * ref.K_EPS
        left_out = ref.calc_output(s.left_g, s.left_h, p, s.l2)
        right_out = ref.calc_output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, p, s.l2)
        node, nl = len(leaves) - 1, len(leaves)
        par = parent_of[pick]
        if par >= 0:
            if T["left_child"][par] == ~pick:
                T["left_child"][par] = node
            else:
                T["right_child"][par] = node
        T["split_feature"].append(s.feature); T["threshold_bin"].append(0 if s.is_cat else s.threshold)
        T["default_left"].append(bool(s.default_left)); T["is_cat"].append(s.is_cat); T["cat_bins"].append(s.cat_bins)
        T["split_gain"].append(float(np.float32(s.gain + p.min_gain_to_split)))
        T["left_child"].append(~pick); T["right_child"].append(~nl)
        T["internal_value"].append(L["value"]); T["internal_weight"].append(L["weight"]); T["internal_count"].append(L["count"])
        lrows, rrows = L["rows"][left], L["rows"][~left]
        flags = dict(L["flags"])
        R = dict(rows=rrows, sum_g=L["sum_g"] - s.left_g, sum_h=sum_h2 - s.left_h - ref.K_EPS, count=len(rrows), best=None,
                 value=0.0 if math.isnan(right_out) else right_out, weight=sum_h2 - s.left_h - ref.K_EPS, flags=dict(flags))
        L.update(rows=lrows, sum_g=s.left_g, sum_h=s.left_h - ref.K_EPS, count=len(lrows), best=None,
                 value=0.0 if math.isnan(left_out) else left_out, weight=s.left_h - ref.K_EPS, flags=flags)
        leaves.append(R)
        parent_of[pick] = node
        parent_of.append(node)
        new_leaves = [pick, nl]
    T["num_leaves"] = len(leaves)
    T["leaf_value"] = [L["value"] if abs(L["value"]) > ref.K_ZERO else 0.0 for L in leaves]
    T["leaf_weight"] = [L["weight"] for L in leaves]
    T["leaf_count"] = [L["count"] for L in leaves]
    T["internal_value"] = [v if abs(v) > ref.K_ZERO else 0.0 for v in T["internal_value"]]
    T["rounds"], T["picks"], T["scanned_counts"] = rounds, picks, []
    return T
