"""NumPy restatement of LightGBM 3.2's monotone constraints with the `basic` method (`monotone_constraints`, `monotone_penalty`) on top of
split_scan_ref.py, and of extra_trees_ref.py for the combined case, used to pin the engine's kMono scans (k_scan, k_scan_wide), the pick
step's clamped outputs and the round controller's leaf bounds tree by tree.

Restated from LightGBM 3.2 (FeatureHistogram's USE_MC branch, BasicLeafConstraints, SerialTreeLearner); not checked against the native
library:
- A non-empty constraint list runs the constrained scans for every feature, even when every entry is 0.
- Every leaf carries bounds [min, max], the root (-inf, +inf).  After a split both children inherit the parent's bounds; a numerical
  split on a monotone feature narrows them at mid = (left_output + right_output) / 2: for +1 the left child's max and the right child's
  min, for -1 the mirror.  Categorical splits never narrow them.
- A candidate's child outputs are CalculateSplittedLeafOutput clamped to the leaf's bounds (after max_delta_step; many-vs-many with
  lambda_l2 + cat_l2); its gain is GetLeafGainGivenOutput(left) + GetLeafGainGivenOutput(right) at those outputs, and 0 when the outputs
  break the split feature's direction.  min_gain_shift stays the leaf's unconstrained GetLeafGain.  The leaf values are the clamped outputs.
- A monotone feature's shifted gain (best gain - min_gain_shift) is multiplied by penalty_factor(depth of the leaf, monotone_penalty)
  before the argmax over features.

The constrained scans re-score split_scan_ref's candidates: those are every candidate that passed the count and hessian tests before a
pass ended, which do not depend on the constraint."""
import math

import numpy as np

import extra_trees_ref as X3
import split_scan_ref as ref

K_EPS_F = float(np.float32(1e-15))      # LightGBM's kEpsilon = 1e-15f, as a double


def clamp(x, lo, hi):
    if x < lo:
        return lo
    if x > hi:
        return hi
    return x


def constrained_output(g, h, p, l2, lo, hi):
    """CalculateSplittedLeafOutput<USE_MC>: max_delta_step first, then the leaf's bounds"""
    return clamp(ref.calc_output(g, h, p, l2), lo, hi)


def gain_given_output(g, h, p, l2, out):
    """GetLeafGainGivenOutput"""
    sg = ref._threshold_l1(g, p.lambda_l1) if p.lambda_l1 > 0 else g
    return -(2.0 * sg * out + (h + l2) * out * out)


def split_gain(lg, lh, rg, rh, p, l2, lo, hi, mono):
    """GetSplitGains<USE_MC>: 0 when the clamped outputs break the direction `mono`"""
    lo_out, ro_out = constrained_output(lg, lh, p, l2, lo, hi), constrained_output(rg, rh, p, l2, lo, hi)
    if (mono > 0 and lo_out > ro_out) or (mono < 0 and lo_out < ro_out):
        return 0.0
    return gain_given_output(lg, lh, p, l2, lo_out) + gain_given_output(rg, rh, p, l2, ro_out)


def penalty_factor(depth, penalty):
    """ComputeMonotoneSplitGainPenalty"""
    if penalty >= depth + 1.0:
        return K_EPS_F
    if penalty <= 1.0:
        return 1.0 - penalty / 2.0 ** depth + K_EPS_F
    return 1.0 - 2.0 ** (penalty - 1.0 - depth) + K_EPS_F


def child_bounds(bounds, mono, is_cat, left_out, right_out):
    """BasicLeafConstraints::Update: (left child's bounds, right child's bounds)"""
    (lo, hi) = bounds
    left, right = [lo, hi], [lo, hi]
    if mono != 0 and not is_cat:
        mid = (left_out + right_out) / 2.0
        if mono > 0:
            left[1], right[0] = min(left[1], mid), max(right[0], mid)
        else:
            left[0], right[1] = max(left[0], mid), min(right[1], mid)
    return tuple(left), tuple(right)


def _rescore(r, p, bounds, mono, keep=None):
    """r's candidates with constrained gains (only those whose tag `keep` accepts); the first strict maximum above min_gain_shift"""
    lo, hi = bounds
    cands = [(split_gain(c[1], c[2], c[3], c[4], p, r.l2, lo, hi, mono),) + tuple(c[1:]) for c in r.candidates if keep is None or keep(c[5])]
    return X3._keep(r, cands)


def find_best_numerical(hg, hh, num_bin, missing_type, offset, sum_g, sum_h_in, num_data, p, feature, bounds, mono, rand_threshold=None):
    r = ref.find_best_numerical(hg, hh, num_bin, missing_type, offset, sum_g, sum_h_in, num_data, p, feature)
    keep = None if rand_threshold is None else (lambda tag: tag[1] == rand_threshold)
    best = _rescore(r, p, bounds, mono, keep)
    two_way = num_bin > 2 and missing_type == 2
    na = 1 if two_way else 0
    r.threshold, r.default_left, r.left_g, r.left_h, r.left_count = 0, True, 0.0, 0.0, 0
    if best is not None:
        cnt = X3._counts(hh, num_bin, sum_h_in, num_data)
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


def find_best_categorical(hg, hh, num_bin, sum_g, sum_h_in, num_data, p, feature, bounds, rand_threshold=None):
    """categorical features carry no constraint of their own (direction 0), but their outputs are clamped to the leaf's bounds"""
    r = ref.find_best_categorical(hg, hh, num_bin, sum_g, sum_h_in, num_data, p, feature)
    onehot = num_bin <= p.max_cat_to_onehot
    keep = None
    if rand_threshold is not None:
        want = {("onehot", rand_threshold + 1)} if onehot else {("dir+1", rand_threshold), ("dir-1", rand_threshold)}
        keep = lambda tag: tag in want      # noqa: E731
    best = _rescore(r, p, bounds, 0, keep)
    cnt = X3._counts(hh, num_bin, sum_h_in, num_data)
    r.cat_bins, r.left_g, r.left_h, r.left_count = (), 0.0, 0.0, 0
    if best is not None:
        if onehot:
            b = best[5][1]
            r.cat_bins, r.left_count = (b,), cnt[b]
        else:
            used = [b for b in range(1, num_bin) if cnt[b] >= p.cat_smooth]
            order = sorted(used, key=lambda b: (float(hg[b]) / (float(hh[b]) + p.cat_smooth), b))
            seq = order if best[5][0] == "dir+1" else order[::-1]
            bins = seq[:best[5][1] + 1]
            r.cat_bins, r.left_count = tuple(sorted(bins)), sum(cnt[b] for b in bins)
        r.left_g, r.left_h = best[1], best[2]
    return r


def _penalise(r, factor):
    """the shifted gain times `factor`.  The candidates keep their own gains: split_scan_ref.undecided compares those with min_gain_shift,
    which the scan does before the penalty; within a leaf every monotone feature has the same factor."""
    if r.gain != ref.NEG_INF:
        r.gain *= factor


def scan_leaf(bins, g, h, rows, leaf, features, p, mono, penalty, streams=None, used=None):
    """split_scan_ref.scan_leaf with the constrained scans at the leaf's bounds and depth; with `streams`, one draw per scanned feature"""
    out = {}
    for f in features:
        if (used is not None and f.real_index not in used) or not leaf["flags"][f.real_index]:
            continue
        col = bins[rows, f.real_index].astype(np.int64)
        hg = np.bincount(col, weights=g[rows], minlength=f.num_bin)
        hh = np.bincount(col, weights=h[rows], minlength=f.num_bin)
        args = (leaf["sum_g"], leaf["sum_h"], leaf["count"], p, f.real_index, leaf["bounds"])
        if f.is_cat:
            t = None if streams is None else streams.draw(f, X3.categorical_range(hh, f.num_bin, leaf["sum_h"], leaf["count"], p))
            out[f.real_index] = find_best_categorical(hg, hh, f.num_bin, *args, rand_threshold=t)
        else:
            t = None if streams is None else streams.draw(f, X3.numerical_range(f.num_bin))
            m = mono[f.real_index]
            out[f.real_index] = find_best_numerical(hg, hh, f.num_bin, f.missing_type, f.offset, *args, m, rand_threshold=t)
            if m != 0:
                _penalise(out[f.real_index], penalty_factor(leaf["depth"], penalty))
    return out


def grow_tree(bins, g, h, features, p, num_leaves, mono, penalty=0.0, extra_trees=False, extra_seed=6, streams=None, used=None):
    """split_scan_ref.grow_tree (extra_trees_ref.grow_tree with extra_trees) under monotone constraints.  mono: the constraint list,
    indexed by real feature (non-empty); the other arguments as extra_trees_ref.grow_tree's.  T["bounds"]: every leaf's final bounds."""
    features = sorted(features, key=lambda f: f.real_index)
    if extra_trees and streams is None:
        streams = X3.Streams(features, extra_seed)
    if not extra_trees:
        streams = None
    used = {f.real_index for f in features} if used is None else set(used)
    n = len(g)
    by_real = {f.real_index: f for f in features}
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags={f.real_index: f.real_index in used for f in features}, bounds=(-math.inf, math.inf), depth=0)]
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
                new_leaves = new_leaves[::-1]            # smaller first (the extra-trees draw order)
            rnd = []
            for l in new_leaves:
                L = leaves[l]
                scans = scan_leaf(bins, g, h, L["rows"], L, features, p, mono, penalty, streams, used)
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
        lo, hi = L["bounds"]
        left_out = constrained_output(s.left_g, s.left_h, p, s.l2, lo, hi)
        right_out = constrained_output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, p, s.l2, lo, hi)
        lb, rb = child_bounds(L["bounds"], 0 if s.is_cat else mono[s.feature], s.is_cat, left_out, right_out)
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
                 value=0.0 if math.isnan(right_out) else right_out, weight=sum_h2 - s.left_h - ref.K_EPS, flags=dict(flags), bounds=rb,
                 depth=L["depth"] + 1)
        L.update(rows=lrows, sum_g=s.left_g, sum_h=s.left_h - ref.K_EPS, count=len(lrows), best=None,
                 value=0.0 if math.isnan(left_out) else left_out, weight=s.left_h - ref.K_EPS, flags=flags, bounds=lb, depth=L["depth"] + 1)
        leaves.append(R)
        parent_of[pick] = node
        parent_of.append(node)
        new_leaves = [pick, nl]
    T["num_leaves"] = len(leaves)
    T["leaf_value"] = [L["value"] if abs(L["value"]) > ref.K_ZERO else 0.0 for L in leaves]
    T["leaf_weight"] = [L["weight"] for L in leaves]
    T["leaf_count"] = [L["count"] for L in leaves]
    T["internal_value"] = [v if abs(v) > ref.K_ZERO else 0.0 for v in T["internal_value"]]
    T["bounds"] = [L["bounds"] for L in leaves]
    T["rounds"], T["picks"], T["scanned_counts"] = rounds, picks, []
    return T
