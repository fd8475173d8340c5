"""NumPy restatement of LightGBM 3.2's path smoothing (`path_smooth`) on top of split_scan_ref.py, monotone_ref.py and extra_trees_ref.py,
used to pin the engine's output-based scans (k_scan, k_scan_wide with kMono), the pick step's smoothed outputs and the leaves' parent
outputs tree by tree.  grow_tree below grows the smoothed trees: tree_ref.grow_tree's rounds and options (voting excepted), with every
leaf's output carried as its children's parent output.

Restated from LightGBM 3.2 (FeatureHistogram's USE_SMOOTHING branch, SerialTreeLearner, Config::CheckParamConflict); not checked against
the native library:
- Smoothing is on when path_smooth > kEpsilon (1e-15f).  With s = path_smooth, a leaf of n rows has the output of
  CalculateSplittedLeafOutput (L1, l2, max_delta_step), then ret * (n/s) / (n/s + 1) + parent_output / (n/s + 1), then, with monotone
  constraints, the leaf's bounds.
- A candidate's gain is GetLeafGainGivenOutput at each child's smoothed (and clamped) output, with the counts the scan estimates:
  RoundInt(h * cnt_factor) summed on one side, num_data minus that on the other.  Many-vs-many uses lambda_l2 + cat_l2.
- min_gain_shift is GetLeafGain<USE_SMOOTHING> of the leaf's own sums and count, smoothed toward parent_output and never clamped, plus
  min_gain_to_split.
- A leaf's parent_output is its own output, the one it got when its parent split.  The root's is its unsmoothed output from its sums
  (without the scans' 2 kEpsilon), so smoothing the root toward it gives it back.
- Leaf and internal values are the smoothed outputs.
- min_data_in_leaf < 2 is raised to 2 when smoothing is on.

The smoothed scans re-score split_scan_ref's candidates, as monotone_ref does: those are every candidate that passed the count and hessian
tests before a pass ended, which do not depend on smoothing."""
import math

import numpy as np

import extra_trees_ref as X3
import interaction_ref as I
import monotone_ref as M
import split_scan_ref as ref
import tree_ref

K_EPS_F = M.K_EPS_F
NO_BOUNDS = (float("-inf"), float("inf"))


def active(s):
    return s > K_EPS_F


def min_data_in_leaf(s, min_data):
    """Config::CheckParamConflict"""
    return 2 if active(s) and min_data < 2 else min_data


def smoothed_output(g, h, n, parent, p, l2, s):
    """CalculateSplittedLeafOutput<USE_SMOOTHING>, in upstream's operation order"""
    ret = ref.calc_output(g, h, p, l2)
    if active(s):
        w = n / s
        ret = ret * w / (w + 1) + parent / (w + 1)
    return ret


def output(g, h, n, parent, p, l2, s, lo, hi):
    """CalculateSplittedLeafOutput<USE_MC, USE_SMOOTHING>: smoothed first, then clamped to the leaf's bounds"""
    return M.clamp(smoothed_output(g, h, n, parent, p, l2, s), lo, hi)


def root_output(sum_g, sum_h, p):
    """the root's parent_output: its own unsmoothed, unclamped output"""
    return ref.calc_output(sum_g, sum_h, p, p.lambda_l2)


def leaf_gain(g, h, n, parent, p, l2, s):
    """GetLeafGain<USE_SMOOTHING>"""
    if not active(s):
        return ref.leaf_gain(g, h, p, l2)
    return M.gain_given_output(g, h, p, l2, smoothed_output(g, h, n, parent, p, l2, s))


def split_gain(lg, lh, rg, rh, lc, rc, parent, p, l2, s, lo, hi, mono):
    """GetSplitGains<USE_MC, USE_SMOOTHING>: 0 when the outputs break the direction `mono`"""
    lo_out, ro_out = output(lg, lh, lc, parent, p, l2, s, lo, hi), output(rg, rh, rc, parent, p, l2, s, lo, hi)
    if (mono > 0 and lo_out > ro_out) or (mono < 0 and lo_out < ro_out):
        return 0.0
    return M.gain_given_output(lg, lh, p, l2, lo_out) + M.gain_given_output(rg, rh, p, l2, ro_out)


def _rescore(r, p, s, parent, sum_g, sum_h_in, num_data, bounds, mono, counts, keep):
    """r's candidates (those whose tag `keep` accepts) with smoothed gains at counts(tag) = (first side, second side), against the
    smoothed min_gain_shift; the first strict maximum above it"""
    lo, hi = bounds
    r.shift = leaf_gain(sum_g, sum_h_in + 2 * ref.K_EPS, num_data, parent, p, p.lambda_l2, s) + p.min_gain_to_split
    cands = []
    for c in r.candidates:
        if keep is not None and not keep(c[5]):
            continue
        a, b = counts(c[5])
        cands.append((split_gain(c[1], c[2], c[3], c[4], a, b, parent, p, r.l2, s, lo, hi, mono),) + tuple(c[1:]))
    return X3._keep(r, cands)


def find_best_numerical(hg, hh, num_bin, missing_type, offset, sum_g, sum_h_in, num_data, p, feature, s, parent, bounds=NO_BOUNDS, mono=0,
                        rand_threshold=None):
    r = ref.find_best_numerical(hg, hh, num_bin, missing_type, offset, sum_g, sum_h_in, num_data, p, feature)
    cnt = X3._counts(hh, num_bin, sum_h_in, num_data)
    two_way = num_bin > 2 and missing_type == 2
    na = 1 if two_way else 0
    base_c = num_data - sum(cnt[1:num_bin]) if offset == 1 else 0

    def left_count(tag):
        kind, t = tag
        return num_data - sum(cnt[t + 1:num_bin - na]) if kind == "rev" else base_c + sum(cnt[offset:t + 1])

    def counts(tag):
        lc = left_count(tag)
        return lc, num_data - lc

    keep = None if rand_threshold is None else (lambda tag: tag[1] == rand_threshold)
    best = _rescore(r, p, s, parent, sum_g, sum_h_in, num_data, bounds, mono, counts, keep)
    r.threshold, r.default_left, r.left_g, r.left_h, r.left_count = 0, True, 0.0, 0.0, 0
    if best is not None:
        r.threshold, r.left_g, r.left_h, r.left_count = best[5][1], best[1], best[2], left_count(best[5])
        r.default_left = best[5][0] == "rev"
    if not two_way and missing_type == 2:
        r.default_left = False
    return r


def find_best_categorical(hg, hh, num_bin, sum_g, sum_h_in, num_data, p, feature, s, parent, bounds=NO_BOUNDS, rand_threshold=None):
    r = ref.find_best_categorical(hg, hh, num_bin, sum_g, sum_h_in, num_data, p, feature)
    onehot = num_bin <= p.max_cat_to_onehot
    cnt = X3._counts(hh, num_bin, sum_h_in, num_data)
    used = [b for b in range(1, num_bin) if cnt[b] >= p.cat_smooth]
    order = sorted(used, key=lambda b: (float(hg[b]) / (float(hh[b]) + p.cat_smooth), b))

    def bins_of(tag):
        if onehot:
            return (tag[1],)
        return tuple((order if tag[0] == "dir+1" else order[::-1])[:tag[1] + 1])

    def counts(tag):
        lc = sum(cnt[b] for b in bins_of(tag))      # one-hot: the candidate's first side is the category's
        return lc, num_data - lc

    keep = None
    if rand_threshold is not None:
        want = {("onehot", rand_threshold + 1)} if onehot else {("dir+1", rand_threshold), ("dir-1", rand_threshold)}
        keep = lambda tag: tag in want      # noqa: E731
    best = _rescore(r, p, s, parent, sum_g, sum_h_in, num_data, bounds, 0, counts, keep)
    r.cat_bins, r.left_g, r.left_h, r.left_count = (), 0.0, 0.0, 0
    if best is not None:
        r.cat_bins = tuple(sorted(bins_of(best[5])))
        r.left_g, r.left_h, r.left_count = best[1], best[2], counts(best[5])[0]
    return r


def scan_leaf(bins, g, h, rows, sum_g, sum_h, num_data, features, flags, p, streams, mono, penalty, bounds, depth, smooth, parent_output):
    """tree_ref.scan_leaf, with the smoothed scans toward parent_output when `smooth` is above kEpsilon (constrained too with a `mono`
    list, a monotone feature's shifted gain times the penalty factor at the leaf's depth); tree_ref.scan_leaf itself otherwise"""
    if not active(smooth):
        return tree_ref.scan_leaf(bins, g, h, rows, sum_g, sum_h, num_data, features, flags, p, streams, mono, penalty, bounds, depth)
    out = {}
    for f in features:
        fi = f.real_index
        if not flags[fi]:
            continue
        col = bins[rows, fi].astype(np.int64)
        hg = np.bincount(col, weights=g[rows], minlength=f.num_bin)
        hh = np.bincount(col, weights=h[rows], minlength=f.num_bin)
        if f.is_cat:
            t = None if streams is None else streams.draw(f, X3.categorical_range(hh, f.num_bin, sum_h, num_data, p))
            out[fi] = find_best_categorical(hg, hh, f.num_bin, sum_g, sum_h, num_data, p, fi, smooth, parent_output, bounds, t)
        else:
            t = None if streams is None else streams.draw(f, X3.numerical_range(f.num_bin))
            m = 0 if mono is None else mono[fi]
            s = out[fi] = find_best_numerical(hg, hh, f.num_bin, f.missing_type, f.offset, sum_g, sum_h, num_data, p, fi, smooth,
                                              parent_output, bounds, m, t)
            if m != 0 and s.gain != ref.NEG_INF:
                s.gain *= M.penalty_factor(depth, penalty)
    return out


def grow_tree(bins, g, h, features, p, num_leaves, *, smooth=0.0, used=None, streams=None, mono=None, penalty=0.0, constraints=None,
              sampler=None, max_depth=-1):
    """One tree as tree_ref.grow_tree grows it with the same options (voting excepted), and with path_smooth = `smooth`: every leaf
    keeps its output, the root its own unsmoothed one (root_output), and the scans and the children's outputs of a leaf are smoothed
    toward it, the outputs with the split's estimated counts.  At or below kEpsilon this is tree_ref.grow_tree's tree, key for key.
    Returns tree_ref.grow_tree's keys."""
    features = sorted(features, key=lambda f: f.real_index)
    by_real = {f.real_index: f for f in features}
    before = sampler.rnd.draws if sampler is not None else 0
    if sampler is not None:
        assert used is None
        used = sampler.by_tree()
    used = set(by_real) if used is None else set(used)
    sets = I.sets_of(constraints if constraints is not None else [list(by_real)], max(by_real) + 1)
    n = len(g)
    leaves = [dict(rows=np.arange(n), sum_g=math.fsum(g), sum_h=math.fsum(h), count=n, best=None, value=0.0, weight=0.0,
                   flags={fi: fi in used for fi in by_real}, bounds=tree_ref.NO_BOUNDS, depth=0, mask=I.ALL, branch=())]
    leaves[0]["output"] = root_output(leaves[0]["sum_g"], leaves[0]["sum_h"], p)
    T = dict(split_feature=[], threshold_bin=[], default_left=[], is_cat=[], cat_bins=[], split_gain=[], left_child=[], right_child=[],
             internal_value=[], internal_weight=[], internal_count=[], rounds=[], picks=[], scanned_counts=[], scan_masks=[],
             node_rounds=[], voted=[])
    parent_of = [-1]
    new_leaves = [0]
    while True:
        counts = [leaves[l]["count"] for l in new_leaves]
        go = len(leaves) < num_leaves and not all(c < p.min_data_in_leaf * 2 for c in counts)
        if go and max_depth > 0 and leaves[new_leaves[0]]["depth"] >= max_depth:
            go = False
        if go:
            T["scanned_counts"].append(list(zip(new_leaves, counts)))
            if len(new_leaves) == 2 and not counts[0] < counts[1]:
                new_leaves = new_leaves[::-1]            # smaller first
            rnd, samples = [], []
            for l in new_leaves:
                L = leaves[l]
                scans = scan_leaf(bins, g, h, L["rows"], L["sum_g"], L["sum_h"], L["count"], features, L["flags"], p, streams, mono,
                                  penalty, L["bounds"], L["depth"], smooth, L["output"])
                for fi, s in scans.items():
                    L["flags"][fi] = s.splittable
                allowed = {fi: s for fi, s in scans.items() if sets[fi] & L["mask"]}
                if sampler is not None:
                    sample = sampler.by_node({fi for fi in sampler.tree if sets[fi] & L["mask"]})
                    samples.append((L["mask"], sample))
                    allowed = {fi: s for fi, s in allowed.items() if fi in sample}
                L["best"] = ref.best_of_leaf(allowed)
                rnd.append((l, L, scans))
            T["rounds"].append(rnd)
            T["scan_masks"].append([leaves[l]["mask"] for l in new_leaves])
            if sampler is not None:
                T["node_rounds"].append(samples)
        else:
            for l in new_leaves:
                leaves[l]["best"] = None
        if len(leaves) >= num_leaves:
            break
        T["picks"].append([(li, L["best"]) for li, L in enumerate(leaves) if L["best"] is not None])
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
        if active(smooth):      # the split's estimated counts, as the pick step has them
            left_out = output(s.left_g, s.left_h, s.left_count, L["output"], p, s.l2, smooth, lo, hi)
            right_out = output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, L["count"] - s.left_count, L["output"], p, s.l2, smooth, lo, hi)
        else:
            left_out = M.constrained_output(s.left_g, s.left_h, p, s.l2, lo, hi)
            right_out = M.constrained_output(L["sum_g"] - s.left_g, sum_h2 - s.left_h, p, s.l2, lo, hi)
        lb, rb = M.child_bounds(L["bounds"], 0 if mono is None or s.is_cat else mono[s.feature], s.is_cat, left_out, right_out)
        mask, branch = L["mask"] & sets[s.feature], L["branch"] + (s.feature,)
        lrows, rrows = L["rows"][left], L["rows"][~left]
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
        flags = dict(L["flags"])
        R = dict(rows=rrows, sum_g=L["sum_g"] - s.left_g, sum_h=sum_h2 - s.left_h - ref.K_EPS, count=len(rrows), best=None,
                 value=0.0 if math.isnan(right_out) else right_out, weight=sum_h2 - s.left_h - ref.K_EPS, flags=dict(flags),
                 bounds=rb, depth=L["depth"] + 1, mask=mask, branch=branch, output=right_out)
        L.update(rows=lrows, sum_g=s.left_g, sum_h=s.left_h - ref.K_EPS, count=len(lrows), best=None,
                 value=0.0 if math.isnan(left_out) else left_out, weight=s.left_h - ref.K_EPS, flags=flags, bounds=lb, depth=L["depth"] + 1,
                 mask=mask, branch=branch, output=left_out)
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
    T["masks"] = [L["mask"] for L in leaves]
    T["branches"] = [L["branch"] for L in leaves]
    T["draws"] = sampler.rnd.draws - before if sampler is not None else 0
    return T
