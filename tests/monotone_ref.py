"""NumPy restatement of LightGBM 3.2's monotone constraints with the `basic` method (`monotone_constraints`, `monotone_penalty`) on top of
split_scan_ref.py and extra_trees_ref.py, the rule tree_ref.grow_tree applies with `mono`, used to pin the engine's kMono scans (k_scan,
k_scan_wide), the pick step's clamped outputs and the round controller's leaf bounds tree by tree.

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
