"""NumPy restatement of LightGBM 3.2's extremely randomised trees (`extra_trees`, `extra_seed`) on top of split_scan_ref.py, the rule
tree_ref.grow_tree applies with `streams`, used to pin the engine's scans (k_scan, k_scan_wide with kExtra) tree by tree and tree after
tree.

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
    """the per-feature Random of every used feature, numbered in real-index order"""

    def __init__(self, features, extra_seed):
        self.rand = {f.real_index: Random(extra_seed + i) for i, f in enumerate(sorted(features, key=lambda f: f.real_index))}

    def draw(self, f, rng):
        return self.rand[f.real_index].next_int(0, rng) if rng > 0 else 0
